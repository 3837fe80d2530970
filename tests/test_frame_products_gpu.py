"""The frame products (DESIGN §8: `frame_products_kernel` and `disparity_image_kernel` of csrc/nfb_post.cu) against the
reference's own functions — torch_normal_map(clean=True), cast_to_image and cast_to_disparity_image of the unmodified
eval_transformed_rays.py, loaded from the staged copy (oracle/stage_reference.py) — run on the same FP32 inputs twice: on torch
CUDA tensors (the kernel's default rounding) and on torch CPU tensors (NFB_PRODUCTS_LIKE_TORCH_CPU).  Every byte of every pixel
must be equal, no tolerance, at:
  sizes        square H = 2 (one normal), 3, 17, 64, 97, 512 and 1024 (past one grid-stride sweep of the 148*8 x 256-thread
               grid); rectangular 64x128, 129x64 and 3x1024 through the C API (rgb and disparity; normals there are
               NFB_ERR_UNSUPPORTED), with the dataset's intrinsics, seeded random ones, and centres whose intr[2] * H is not an FP32
  disparity    one NaN, all NaN, a NaN made on the GPU as 0/0 and a sign-bit-set NaN (-float('nan')), both kinds together; +inf,
               -inf, both, all inf; constant frames, constant but one pixel; -0.0 beside +0.0; negative frames; subnormal values;
               tiny (1e-17, 1e-20) values whose normals come out +-inf; the renderer's 1/1e-10 cap; a range that overflows to inf
  normals      flat patches (zero disparity: a zero cross product, 0/0), NaN disparities beside valid ones, with the cleaning
               mask w_last cycling over {0, 0.22f - ulp, 0.22f, 0.22f + ulp, 1, NaN} and with w_last = None
  rgb          every k / 255 (both FP32 roundings of it) and its FP32 neighbours, below 0, above 1, +-0, NaN, +-inf
  call shapes  rgb only, disparity only, normals without the disparity image; two calls in a row on one handle and stream,
               the second frame's disparity range strictly inside the first's (the handle's one min / max scratch)
  end to end   render_camera (both precisions) of a frame whose fine network's sigma output puts about half of it in empty
               space, with NaN and inf background pixels; the kernel's own rgb_fine, disp_fine and w_last fed to both sides.

Empty space is not 0/0.  The reference adds 1e-6 to the last sample's sigma and gives that sample a 1e10 gap, so a ray whose
every sigma is 0 is stopped by its last sample: alpha = 1 - exp(-1e4 |d|) = 1, w_last = 1, acc = 1 and disp = 1 / far.  The
end-to-end case asserts exactly that for those pixels; NaN disparities reach the products only from NaN inputs, and are tested
directly above.

What the reference's bytes are for NaN and out-of-range values is decided by its last, host-side conversion
(`.cpu().numpy().astype("uint8")`, and torchvision's `.mul(255).byte()` on a CPU tensor).  On the x86-64 host these tests ran
on (numpy 2.3, torch 2.11) both truncate to int32 and keep the low byte, so NaN, +inf and -inf all become 0 (and 256 -> 0,
-1 -> 255).  `cast_to_disparity_image` of a frame holding any NaN is therefore all 0 (torch's min / max propagate NaN), as is a
pixel whose normalised value is inf / inf.  These tests rely on the GPU machine's host converting the same way; the kernel's
to_u8 reproduces it.

What these tests found (both fixed in csrc/nfb_post.cu):
  * to_u8 converted with the device's saturating float -> int, so a +inf normal component became 255 where the reference has
    0: test_disparity_edges[tiny_1e-17, tiny_1e-20, subnormal_and_normal], both modes.
  * torch CUDA divides by fx as a multiplication by fp32(1 / fx) with the reciprocal taken in double; the kernel used
    1 / fp32(fx), which differs when fx is not an FP32 (the dataset's 1200 * H / 512 always is): one byte off at up to 1,374
    of 1,046,529 normals, test_square_frames[97 / 512 unrepresentable_centre, 1024 random] in CUDA mode.
  test_post_gpu.py's golden comparison (dataset intrinsics, disparities in [1, 5]) passes with either defect.

Planted defects, each built once in a copy of the source and not kept; what fails here, and whether test_post_gpu.py does:
  (a) no min / max reset in launch_frame_products: every case with a disparity image; test_post_gpu.py fails too.
  (b) `>=` instead of `>` at 0.22: test_normal_edges, both modes; test_post_gpu.py passes.
  (c) the CPU order of the squared sum in CUDA mode: test_square_frames at 512 and 1024 (CUDA mode); test_post_gpu.py fails
      too.
  (d) the clamps as fmaxf(fminf(v, 1), 0): nvcc (12.9, -O3) compiles both orders to one saturating add (FADD.SAT, NaN -> 0),
      so this changes no byte and no test can see it.  What the order means in C (NaN -> 1), planted as an explicit
      `isnan(v) ? 1 : ...` in both clamps: test_rgb_edges and every NaN disparity case, both modes; test_post_gpu.py passes.
  (e) the min key taken from fabsf of the value: the negative, -inf, negative-NaN and overflowing-range disparity cases and
      the two C API tests, both modes; test_post_gpu.py passes.
  The parent's two rules found above were run the same way: each fails only the cases named with it.

Measured on an H100 80GB HBM3 at a 700 W power limit: the 106 cases take about 21 s, 11 s of it the first setup (build
check, reference import, handle); a 1024x1024 case takes 0.11 to 0.23 s, most of it the torch reference.
"""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import nerface_oracle as O
import ref_loader

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(ref_loader.reference_root(staged_only=True) is None,
                                 reason="no staged reference in oracle/_ref (build() stages it; oracle/stage_reference.py)")]

NEAR, FAR = 0.2, 0.8
MODES = ["cuda", "cpu"]          # which torch back end runs the reference; the kernel follows it (like_torch_cpu)
F32 = np.float32


@pytest.fixture(scope="module")
def P(built_lib):
    import nerf
    from nerf import _capi, _engine, ray_sampler
    ev = ref_loader.load_eval_script(staged_only=True)
    assert ev is not None
    dev = torch.device("cuda", 0)
    return types.SimpleNamespace(nerf=nerf, capi=_capi, engine=_engine, ray_sampler=ray_sampler, ev=ev, dev=dev,
                                 eng=_engine.renderer_for(dev))


# ------------------------------------------------------------------------------------------------ the two sides
def reference_products(P, mode, c, d, w, intr, normals=True):
    """The reference functions exactly as the eval script (and oracle/make_golden_live.py::gen_products_cuda) call them, on
    tensors of the back end `mode`.  Returns numpy uint8 (rgb [H,W,3], normals [H-1,W-1,3] or None, disparity [H,W])."""
    dev = P.dev if mode == "cuda" else torch.device("cpu")
    c, d = c.to(dev), d.to(dev)
    w = w.to(dev) if w is not None else None
    with np.errstate(invalid="ignore"):  # NaN / inf -> uint8 (see the module docstring)
        n = None
        if normals:
            n = P.ev.torch_normal_map(d.clone(), intr, w.clone() if w is not None else None, clean=True).cpu().numpy().astype("uint8")
        disp = np.asarray(P.ev.cast_to_disparity_image(d))
        rgb = np.asarray(P.ev.cast_to_image(c, "blender"))
    return rgb, n, disp


def kernel_products(P, mode, c, d, w, intr):
    rgb, n, disp = P.ray_sampler.frame_products(c.to(P.dev), d.to(P.dev), w.to(P.dev) if w is not None else None, list(intr),
                                                want_disparity=True, like_torch_cpu=mode == "cpu")
    return rgb.cpu().numpy(), n.cpu().numpy(), disp.cpu().numpy()


def capi_products(P, c, d, w, intr, H, W, rgb=True, normals=True, disparity=True, like_cpu=False, check=True):
    """nfb_frame_products with only the requested outputs (the rest NULL), into buffers pre-filled with a poison byte."""
    def buf(shape, want):
        return torch.full(shape, 0xA5, dtype=torch.uint8, device=P.dev) if want else None
    o_rgb, o_n, o_d = buf((H, W, 3), rgb), buf((H - 1, W - 1, 3), normals), buf((H, W), disparity)
    ptr = P.engine._ptr
    dev_or_none = lambda t: t.to(P.dev).contiguous() if t is not None else None  # noqa: E731
    c, d, w = dev_or_none(c), dev_or_none(d), dev_or_none(w)
    rc = P.capi.lib.nfb_frame_products(P.eng._h, ptr(c), ptr(d), ptr(w), (C.c_double * 4)(*[float(v) for v in intr]), H, W,
                                       ptr(o_rgb), ptr(o_n), ptr(o_d), 1 if like_cpu else 0,  # NFB_PRODUCTS_LIKE_TORCH_CPU
                                       P.engine._stream())
    if check:
        P.capi.check(rc, "frame_products")
    return rc, o_rgb, o_n, o_d


def assert_bytes_equal(tag, got, want, c, d, w):
    """Exact equality at every pixel; otherwise the count of differing pixels, the worst byte difference and the first differing
    pixel with the inputs it is computed from."""
    got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    assert got.dtype == np.uint8 and got.shape == want.shape, (tag, got.dtype, got.shape, want.shape)
    diff = got != want
    if not diff.any():
        return
    per_pixel = diff.reshape(diff.shape[0], diff.shape[1], -1).any(-1)
    r, q = (int(v) for v in np.argwhere(per_pixel)[0])
    worst = int(np.abs(got.astype(np.int16) - want.astype(np.int16)).max())
    hexf = lambda v: f"{float(v)!r} ({np.asarray(v, dtype=F32).view(np.uint32):#010x})"  # noqa: E731
    if tag.startswith("normals"):
        ins = dict(d00=hexf(d[r, q]), d01=hexf(d[r, q + 1]), d10=hexf(d[r + 1, q]), w=hexf(w[r, q]) if w is not None else None)
    elif tag.startswith("disparity"):
        ins = dict(d=hexf(d[r, q]), min=hexf(d.min()), max=hexf(d.max()), nan=bool(torch.isnan(d).any()))
    else:
        ins = dict(rgb=[hexf(v) for v in c[r, q]])
    pytest.fail(f"{tag}: {int(per_pixel.sum())} of {per_pixel.size} pixels differ, worst byte difference {worst}; first at "
                f"({r}, {q}): kernel {got[r, q].tolist()} reference {want[r, q].tolist()}, inputs {ins}")


def check_frame(P, mode, tag, c, d, w, intr, no_clean_too=True):
    """All three products, and the uncleaned normal map, of one square frame against the reference."""
    c, d = c.float().cpu(), d.float().cpu()
    w = w.float().cpu() if w is not None else None
    want = reference_products(P, mode, c, d, w, intr)
    got = kernel_products(P, mode, c, d, w, intr)
    for name, g, r in zip(("rgb", "normals", "disparity"), got, want):
        assert_bytes_equal(f"{name} [{tag}, {mode}]", g, r, c, d, w)
    if no_clean_too and w is not None:
        _, n_ref, _ = reference_products(P, mode, c, d, None, intr)
        _, n_got, _ = kernel_products(P, mode, c, d, None, intr)
        assert_bytes_equal(f"normals, w_last None [{tag}, {mode}]", n_got, n_ref, c, d, None)


# ------------------------------------------------------------------------------------------------ inputs
def base_frame(H, W, seed):
    """Like oracle/make_golden_live.py::products_inputs: disparity in [1, 5], w_last = U^3, rgb in [-0.1, 1.1]."""
    g = torch.Generator().manual_seed(seed)
    d = torch.rand(H, W, generator=g) * 4 + 1
    w = torch.rand(H, W, generator=g) ** 3
    c = torch.rand(H, W, 3, generator=g) * 1.2 - 0.1
    return c, d, w


def intrinsics(kind, H):
    if kind == "dataset":      # products_inputs
        return np.array([1200.0 * H / 512, 1150.0 * H / 512, 0.52, 0.47])
    rng = np.random.default_rng(1000 + H)
    if kind == "random":
        f = rng.uniform(50.0, 3000.0, 2) * rng.choice([-1.0, 1.0], 2)
        return np.array([f[0], f[1], rng.uniform(0.05, 0.95), rng.uniform(0.05, 0.95)])
    # centres with more significant bits than FP32 keeps: intr[2] * H and intr[3] * H round when they become the FP32 cx, cy
    intr = np.array([rng.uniform(300.0, 2000.0), rng.uniform(300.0, 2000.0), 0.4999999999 + 1e-7 / 3, 1 / 3 + 1e-9])
    assert float(F32(intr[2] * H)) != intr[2] * H and float(F32(intr[3] * H)) != intr[3] * H
    return intr


SQUARE = [2, 3, 17, 64, 97, 512, 1024]
INTRINSICS = ["dataset", "random", "unrepresentable_centre"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", INTRINSICS)
@pytest.mark.parametrize("H", SQUARE)
def test_square_frames(P, H, kind, mode):
    c, d, w = base_frame(H, H, H)
    check_frame(P, mode, f"{H}x{H} {kind}", c, d, w, intrinsics(kind, H))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("H,W", [(64, 128), (129, 64), (3, 1024)])
def test_rectangular_frames(P, H, W, mode):
    """rgb and disparity of H != W frames through the C API; normals there are refused (the reference's expression only
    broadcasts for square frames)."""
    c, d, w = base_frame(H, W, 7 * H + W)
    if H == 129:
        d[H // 2, W // 3] = float("nan")
    intr = intrinsics("random", H)
    rgb_ref, _, disp_ref = reference_products(P, mode, c, d, w, intr, normals=False)
    _, rgb, _, disp = capi_products(P, c, d, w, intr, H, W, normals=False, like_cpu=mode == "cpu")
    assert_bytes_equal(f"rgb [{H}x{W}, {mode}]", rgb, rgb_ref, c, d, w)
    assert_bytes_equal(f"disparity [{H}x{W}, {mode}]", disp, disp_ref, c, d, w)
    rc = capi_products(P, c, d, w, intr, H, W, check=False)[0]
    assert rc == 2  # NFB_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------ disparity edges
def nan_bits(v):
    return int(np.asarray(v, dtype=F32).view(np.uint32))


def neg_nan():
    x = torch.tensor(-float("nan"), dtype=torch.float32)
    assert nan_bits(x) & 0x80000000 and torch.isnan(x)
    return x


def gpu_nan(P):
    z = torch.zeros((), device=P.dev)
    x = (z / z).cpu()                               # 0/0 on the device: the canonical NaN, sign bit clear
    assert torch.isnan(x) and not nan_bits(x) & 0x80000000
    return x


def disparity_case(P, name, d):
    H, W = d.shape
    g = torch.Generator().manual_seed(len(name))
    u = torch.rand(H, W, generator=g)
    cap = float(F32(1.0) / F32(1e-10))              # the renderer's 1 / max(1e-10, depth / acc)
    if name == "one_nan":
        d[5, 7] = float("nan")
    elif name == "all_nan":
        d[:] = float("nan")
    elif name == "gpu_nan_0_over_0":
        d[3, 4] = gpu_nan(P)
    elif name == "negative_nan":
        d[6, 2] = neg_nan()
    elif name == "both_nans":
        d[6, 2], d[H - 1, W - 1] = neg_nan(), gpu_nan(P)
    elif name == "all_negative_nan":
        d[:] = neg_nan()
    elif name == "plus_inf":
        d[2, 9] = math.inf
    elif name == "minus_inf":
        d[8, 1] = -math.inf
    elif name == "both_infs":
        d[2, 9], d[8, 1] = math.inf, -math.inf
    elif name == "all_inf":
        d[:] = math.inf
    elif name == "constant":
        d[:] = 2.5
    elif name == "constant_but_one_above":
        d[:] = 2.5
        d[4, 11] = 3.0
    elif name == "constant_but_one_below":
        d[:] = 2.5
        d[H - 2, 0] = 2.0
    elif name == "signed_zeros":
        d[:] = 0.0
        d[1::2] = -0.0
        d[::3, ::2] = u[::3, ::2]
    elif name == "only_signed_zeros":
        d[:] = 0.0
        d[:, 1::2] = -0.0
    elif name == "negative":
        d[:] = u * 4 - 3
    elif name == "all_negative":
        d[:] = -(u * 4 + 1)
    elif name == "subnormal":
        d[:] = u * 1e-39
        d[0, 0] = 1.4e-45
    elif name == "subnormal_and_normal":
        d[::2] = u[::2] * 1e-40
    elif name == "tiny_1e-17":
        d[:] = (u + 1) * 1e-17
    elif name == "tiny_1e-20":
        d[:] = (u + 1) * 1e-20
    elif name == "cap_1e10":
        d[::4, ::3] = cap
    elif name == "all_at_cap":
        d[:] = cap
    elif name == "range_overflows":
        d[0, 0], d[H - 1, 0] = -3e38, 3e38
    else:
        raise KeyError(name)
    return d


DISPARITY_CASES = ["one_nan", "all_nan", "gpu_nan_0_over_0", "negative_nan", "both_nans", "all_negative_nan", "plus_inf",
                   "minus_inf", "both_infs", "all_inf", "constant", "constant_but_one_above", "constant_but_one_below",
                   "signed_zeros", "only_signed_zeros", "negative", "all_negative", "subnormal", "subnormal_and_normal",
                   "tiny_1e-17", "tiny_1e-20", "cap_1e10", "all_at_cap", "range_overflows"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", DISPARITY_CASES)
def test_disparity_edges(P, case, mode):
    H = 33
    c, d, w = base_frame(H, H, 11)
    d = disparity_case(P, case, d)
    check_frame(P, mode, case, c, d, w, intrinsics("dataset", H))


# ------------------------------------------------------------------------------------------------ normal edges
W_EDGES = [0.0, float(np.nextafter(F32(0.22), F32(0))), float(F32(0.22)), float(np.nextafter(F32(0.22), F32(1))), 1.0,
           float("nan")]


@pytest.mark.parametrize("mode", MODES)
def test_normal_edges(P, mode):
    """Flat patches at zero disparity (a zero cross product: 0/0), NaN disparities among valid ones, and every w_last edge at
    each of them: the mask cycles through W_EDGES along the row-major pixel index, and 41 columns shift the cycle per row."""
    H = 41
    c, d, w = base_frame(H, H, 23)
    d[10:16, 10:16] = 0.0                      # flat: every normal inside and on its top / left border is 0/0
    d[30:34, 2:9] = -0.0
    d[3:8, 20:40] = 2.0                        # constant, not flat: (x, y) still move with the column and row
    idx = torch.arange(H * H).reshape(H, H)
    d[(idx % 7 == 3) & (idx < H * H // 2)] = float("nan")   # isolated NaNs: each spoils three normals
    d[25, :] = float("nan")                                 # a NaN row
    w = torch.tensor(W_EDGES)[idx % len(W_EDGES)]
    assert (w == F32(0.22)).sum() > 100
    check_frame(P, mode, "normal edges", c, d, w, intrinsics("dataset", H))


# ------------------------------------------------------------------------------------------------ rgb edges
def rgb_edge_values():
    k = np.arange(256, dtype=F32)
    on = [k / F32(255), (np.arange(256) / 255.0).astype(F32)]   # both FP32 roundings of k / 255
    vals = []
    for v in on:
        vals += [v, np.nextafter(v, F32(-1)), np.nextafter(v, F32(2))]
    special = np.array([-1.0, -1e-30, -0.0, 0.0, 1.4e-45, 1.0, 1.5, 1e30, 3.4e38, math.inf, -math.inf, math.nan, 0.5], dtype=F32)
    special = np.concatenate([special, neg_nan().numpy().reshape(1)])
    return np.concatenate(vals + [special]).astype(F32)


@pytest.mark.parametrize("mode", MODES)
def test_rgb_edges(P, mode):
    """Every k / 255 and its FP32 neighbours, so that x255 lands on and beside each integer; below 0, above 1, NaN, +-inf."""
    H = 48
    c, d, w = base_frame(H, H, 31)
    v = torch.from_numpy(rgb_edge_values())
    flat = c.reshape(-1)
    flat[:v.numel()] = v
    flat[v.numel():2 * v.numel()] = v.flip(0)      # each value in another channel too
    check_frame(P, mode, "rgb edges", c, d, w, intrinsics("dataset", H), no_clean_too=False)


# ------------------------------------------------------------------------------------------------ call shapes
@pytest.mark.parametrize("mode", MODES)
def test_one_product_per_call(P, mode):
    """rgb only, disparity only, and normals without the disparity image: each NULL output is skipped, the others equal the
    reference."""
    H = 40
    c, d, w = base_frame(H, H, 41)
    d[7, 7] = -2.0
    intr = intrinsics("random", H)
    rgb_ref, n_ref, disp_ref = reference_products(P, mode, c, d, w, intr)
    like_cpu = mode == "cpu"
    _, rgb, _, _ = capi_products(P, c, None, None, intr, H, H, normals=False, disparity=False, like_cpu=like_cpu)
    assert_bytes_equal(f"rgb only [{mode}]", rgb, rgb_ref, c, d, w)
    _, _, _, disp = capi_products(P, None, d, None, intr, H, H, rgb=False, normals=False, like_cpu=like_cpu)
    assert_bytes_equal(f"disparity only [{mode}]", disp, disp_ref, c, d, w)
    _, _, n, _ = capi_products(P, None, d, w, intr, H, H, rgb=False, disparity=False, like_cpu=like_cpu)
    assert_bytes_equal(f"normals only [{mode}]", n, n_ref, c, d, w)


@pytest.mark.parametrize("mode", MODES)
def test_two_calls_in_a_row(P, mode):
    """One handle, one stream, no synchronisation between the calls: the second frame's disparity range lies strictly inside the
    first's, so a min / max left over from the first call would show in every byte of the second disparity image."""
    H = 64
    c1, d1, w1 = base_frame(H, H, 51)
    c2, d2, w2 = base_frame(H, H, 52)
    d1 = d1 * 5 - 15                 # [-10, 10]
    d2 = d2 * 0.5 + 0.5              # [1, 3]
    intr = intrinsics("dataset", H)
    like_cpu = mode == "cpu"
    first = capi_products(P, c1, d1, w1, intr, H, H, like_cpu=like_cpu)[1:]
    second = capi_products(P, c2, d2, w2, intr, H, H, like_cpu=like_cpu)[1:]
    for tag, got, (c, d, w) in (("first", first, (c1, d1, w1)), ("second", second, (c2, d2, w2))):
        want = reference_products(P, mode, c, d, w, intr)
        for name, g, r in zip(("rgb", "normals", "disparity"), got, want):
            assert_bytes_equal(f"{name} [{tag} call, {mode}]", g, r, c, d, w)


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_end_to_end_empty_space(P, prec):
    """render_camera's own rgb_fine, disp_fine and w_last, with part of the frame in empty space, into the products."""
    H = W = 48
    n = H * W
    fr = O.synthetic_frame(31, H, W)
    pc, pf = O.random_init_params(100, True), O.random_init_params(101, True)
    # fine-pass sigma raw = 300 (raw - 10.5): about half the rays get sigma <= 0 at every sample, the rest are dense enough
    # that w_last falls on both sides of 0.22
    pf["fc_alpha.weight"] = pf["fc_alpha.weight"] * 300.0
    pf["fc_alpha.bias"] = (pf["fc_alpha.bias"] - 10.5) * 300.0
    models = []
    for p in (pc, pf):
        m = P.nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                              include_input_xyz=True, include_input_dir=False)
        m.load_state_dict(p)
        models.append(m.to(P.dev))
    P.eng.sync_weights(*models)
    P.eng.set_frame(fr["expr"].to(P.dev), fr["latent"].to(P.dev))
    bg = fr["bg"].reshape(-1, 3).clone()
    bg[::37] = float("nan")
    bg[5::41, 1] = math.inf
    bg = bg.to(P.dev).contiguous()
    v = P.eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, NEAR, FAR, 64, 128, background=bg, precision=prec)
    dbg = P.eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, NEAR, FAR, 64, 128, background=bg, precision=prec,
                              debug=True)
    torch.cuda.synchronize()
    empty = (dbg["raw_fine"][..., 3] <= 0).all(-1)
    assert 0 < int(empty.sum()) < n, int(empty.sum())
    # sigma 0 everywhere but the last sample's 1e-6 over a 1e10 gap: the last sample takes the whole ray
    assert bool((v["acc_fine"][empty] == 1).all()) and bool((v["w_last"][empty] == 1).all())
    assert bool((v["disp_fine"][empty] == float(F32(1) / F32(FAR))).all())
    assert bool(torch.isnan(v["rgb_fine"]).any()) and not bool(torch.isnan(v["disp_fine"]).any())
    c, d, w = v["rgb_fine"].view(H, W, 3), v["disp_fine"].view(H, W), v["w_last"].view(H, W)
    assert bool((w > 0.22).any()) and bool((w <= 0.22).any()), "the cleaning mask takes both sides of 0.22"
    for mode in MODES:
        check_frame(P, mode, f"render {prec}", c.clone(), d.clone(), w.clone(), np.array(fr["intrinsics"]))
