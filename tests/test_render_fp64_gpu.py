"""The evaluation render kernel (render_kernel<*, false>, csrc/nfb_render.cu) against float64, stage by stage, at every tile
of its persistent schedule, and at its FP16-range and non-finite edges.

Each stage is fed the kernel's own output of the stage before, read from the NfbDebug dumps (z_coarse, raw_coarse, z_fine,
raw_fine).  Resampling and sorting are discontinuous, so this keeps every comparison well-posed.  The references are the
existing ones, evaluated in float64 on the GPU: tests/torch_reference._mlp for the MLP, nerface_oracle.composite and
nerface_oracle.resample for compositing and the inverse CDF (both follow their input's dtype).
  (a) coarse depths   bitwise equal to the FP32 formula (separate torch ops), with and without the stratified jitter.
  (b) MLP             raw_coarse / raw_fine against the float64 MLP at the kernel's sample points (formed in FP32 as the
                      kernel forms them, o + d*z rounded separately, then promoted): max-abs / max|ref| and relative L2 per
                      output (rgb raw, sigma raw).  Schedule uniformity: every sample is mapped to its class (CTA iteration
                      0 or >= 1, pass, tile within the unit, warpgroup half, tile ordinal within the CTA mod 10 -- 32 weight
                      units per tile is 2 mod 5, so the mod 10 covers the 5 ring slots at both barrier parities); the worst
                      class's RMS error must stay within KAPPA x the overall RMS.  FP16 rounding noise is the same everywhere
                      in the schedule; a defect in one slot, one iteration or one straddling tile is not.
  (c) compositing     the seven outputs against float64 composite of the kernel's own raw and z (FP32 in both modes).
  (d) resampling      z_fine is non-decreasing, holds every z_coarse value bit for bit (as a multiset), and its remainder,
                      sorted, lies inside the sorted float64 bounds described at resample_bounds().

Measured on an H100 80GB HBM3 at a 400 W power limit (CUDA 12.9), worst over all cases and both passes:
  (b) exact   max 9.6e-6 / L2 1.4e-5 of the channel scale (1024^2 band, coarse sigma)   -> MLP_TOL exact (4e-5, 4e-5)
      fast    max 1.9e-3 / L2 1.3e-3                                                  -> MLP_TOL fast  (6e-3, 4e-3)
      worst class RMS / overall RMS: exact 1.56, fast 1.31                            -> KAPPA 2.5
  (c) max 4.3e-6 of max(1, max|ref|) (random-init weights; 1.1e-6 on opaque ones)    -> COMP_TOL 1.5e-5
  (d) no sample outside its bound.
  FP16 range (exact, activations in (65504, 131008)): 2.3e-5                         -> RANGE_TOL_EXACT_SAT 1e-4
A defect these tests were checked against, each built once: the wrong ray's direction term in step 6's epilogue for
the second row group of a thread (100c+60f: MLP max error 6.4e-3), exact mode skipping the lo MMA on fine tiles t >= 1
(6.4e-4 against 4e-5), and the resampling's den < 1e-5 clamp removed (non-finite fine samples).
"""
import types

import pytest
import torch

import nerface_oracle as O
import torch_reference as TR

pytestmark = pytest.mark.gpu

NEAR, FAR = 0.2, 0.8
NAMES = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
PRECS = ["exact", "fast"]
MLP_TOL = {"exact": (4e-5, 4e-5), "fast": (6e-3, 4e-3)}   # (max-abs / max|ref|, relative L2) per output channel group
KAPPA = 2.5            # worst schedule class RMS error / overall RMS error
CLASS_MIN = 512        # samples a class needs before its RMS counts
COMP_TOL = 1.5e-5        # compositing: max-abs / max(1, max|ref|) per output
U32 = 2.0 ** -24       # unit roundoff of FP32
Z_SLACK = 8 * U32      # FP32 rounding of a bin mid-point and of the interpolation, on depths < 1


@pytest.fixture(scope="module")
def E(built_lib):
    import nerf
    from nerf import _engine
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    e = types.SimpleNamespace(nerf=nerf, dev=torch.device("cuda", 0))
    e.eng = _engine.renderer_for(e.dev)
    e.sms = torch.cuda.get_device_properties(0).multi_processor_count
    fr = O.synthetic_frame(21, 48, 48)
    ro, rd = O.ray_bundle(48, 48, fr["intrinsics"], fr["pose"])
    e.ro, e.rd = ro.reshape(-1, 3).to(e.dev), rd.reshape(-1, 3).to(e.dev)
    e.bg = fr["bg"].reshape(-1, 3).to(e.dev)
    e.expr, e.latent = fr["expr"].to(e.dev), fr["latent"].to(e.dev)
    e._models = {}
    return e


def model(E, seed, stress, params=None):
    key = (seed, stress)
    if params is None and key in E._models:
        return E._models[key]
    m = E.nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                          include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params if params is not None else O.random_init_params(seed, stress))
    m = m.to(E.dev)
    if params is None:
        E._models[key] = m
    return m


def two_iter_rays(E):
    """4 * SMs + 37 rays: with two rays per unit every CTA runs at least two units and the last unit is half filled."""
    return 4 * E.sms + 37


def make_case(E, n, nc, nf, prec, stress=True, perturb=False, noise_std=0.0, bg=True, white=False, dir_z=False, seed=0):
    g = torch.Generator().manual_seed(2000 + seed)
    nz = O.draw_noise(n, O.Sampling(nc, nf, perturb, noise_std, white, 2048), g)
    noise = {k: getattr(nz, k).to(E.dev) for k in ("t_rand", "n_c", "u", "n_f") if getattr(nz, k) is not None}
    idx = torch.arange(n, device=E.dev) % E.ro.shape[0]
    return types.SimpleNamespace(
        n=n, nc=nc, nf=nf, prec=prec, perturb=perturb, noise_std=noise_std, white=white, noise=noise, camera=None,
        ro=E.ro[idx].contiguous(), rd=E.rd[idx].contiguous(), bg=E.bg[idx].contiguous() if bg else None,
        dz=(torch.rand(n, generator=g) * 2.0 - 1.0).to(E.dev) if dir_z else None, expr=E.expr, latent=E.latent,
        mc=model(E, 100, stress), mf=model(E, 101, stress) if nf > 0 else None)


def camera_case(E, H, row_begin, rows, nc, nf, prec):
    """Image rows [row_begin, row_begin + rows) of an H x H frame, rendered with in-kernel ray generation.  The explicit
    rays of the same pixels (nerface_oracle.ray_bundle: the same FP32 operations) serve the reference."""
    fr = O.synthetic_frame(1, H, H)
    ro, rd = O.ray_bundle(H, H, fr["intrinsics"], fr["pose"])
    sl = slice(row_begin * H, (row_begin + rows) * H)
    c = types.SimpleNamespace(
        n=rows * H, nc=nc, nf=nf, prec=prec, perturb=False, noise_std=0.0, white=False, noise={},
        camera=(fr["pose"], fr["intrinsics"], H, row_begin, rows),
        ro=ro.reshape(-1, 3)[sl].contiguous().to(E.dev), rd=rd.reshape(-1, 3)[sl].contiguous().to(E.dev),
        bg=fr["bg"].reshape(-1, 3)[sl].contiguous().to(E.dev), dz=None, expr=fr["expr"].to(E.dev),
        latent=fr["latent"].to(E.dev), mc=model(E, 100, True), mf=model(E, 101, True))
    return c


def render(E, c):
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    if c.camera is not None:
        pose, intr, H, row_begin, rows = c.camera
        out = E.eng.render_camera(pose, intr, H, H, row_begin, rows, NEAR, FAR, c.nc, c.nf, background=c.bg,
                                  precision=c.prec, debug=True)
    else:
        out = E.eng.render(c.ro, c.rd, NEAR, FAR, c.nc, c.nf, perturb=c.perturb, noise_std=c.noise_std, white_bkgd=c.white,
                           background=c.bg, dir_z=c.dz, noise=c.noise or None, precision=c.prec, debug=True)
    torch.cuda.synchronize()
    return out


def schedule(E, c):
    """Rays per unit, tiles per pass and grid, as nfb_render_forward launches the kernel."""
    R = 2 if 2 * (c.nc + c.nf) <= 512 else 1
    tc = (R * c.nc + 127) // 128
    tf = (R * (c.nc + c.nf) + 127) // 128 if c.nf else 0
    n_units = (c.n + R - 1) // R
    return types.SimpleNamespace(R=R, tc=tc, tf=tf, n_units=n_units, grid=min(n_units, E.sms))


def f64(t):
    return None if t is None else t.detach().double()


def params64(m, replace=None):
    p = {k: f64(v) for k, v in m.named_parameters()}
    p.update(replace or {})
    return p


def dir_cols64(c):
    near, far = (torch.tensor(v, dtype=torch.float32).double() for v in (NEAR, FAR))  # the kernel's FP32 near / far
    dz = c.dz if c.dz is not None else c.rd[:, 2]
    return torch.stack((dz.double(), near.expand(c.n).to(dz.device), far.expand(c.n).to(dz.device)), dim=-1)


def mlp64(c, p, z, chunk=1 << 19):
    """float64 MLP output [n, S, 4] at the kernel's depths z [n, S]; sample points formed in FP32 like the kernel's."""
    n, S = z.shape
    pts = (c.ro[:, None, :] + c.rd[:, None, :] * z[:, :, None]).reshape(-1, 3)
    dirs = dir_cols64(c)
    expr, lat = f64(c.expr), f64(c.latent)
    out = torch.empty(n * S, 4, dtype=torch.float64, device=z.device)
    for b in range(0, n * S, chunk):
        e = min(n * S, b + chunk)
        ray = torch.arange(b, e, device=z.device) // S
        x = torch.cat((TR._posenc(pts[b:e].double(), 10, True), TR._posenc(dirs[ray], 4, False)), dim=-1)
        out[b:e] = TR._mlp(p, x, expr, lat)
    return out.view(n, S, 4)


def errors(got, ref):
    """(max-abs error / max |ref|, relative L2 error)."""
    d = got.double() - ref
    return float(d.abs().max() / ref.abs().max()), float(d.norm() / ref.norm())


def sample_classes(E, c, sch, pas):
    """Schedule class of every (ray, sample) of one pass: CTA iteration 0 / >= 1, pass, tile within the unit, warpgroup
    half, tile ordinal within the CTA mod 10."""
    S = c.nc + c.nf if pas else c.nc
    ray = torch.arange(c.n, device=E.dev).view(-1, 1)
    i = torch.arange(S, device=E.dev).view(1, -1)
    unit, rr = ray // sch.R, ray % sch.R
    it = unit // sch.grid
    prow = rr * S + i
    t = prow // 128
    half = (prow % 128) // 64
    ordinal = it * (sch.tc + sch.tf) + (sch.tc if pas else 0) + t
    key = (((it.clamp(max=1) * 2 + pas) * 4 + t) * 2 + half) * 10 + ordinal % 10
    return key.reshape(-1)


def check_uniformity(tag, errs, classes):
    """errs: per-sample squared error of one output channel group; classes: their schedule class."""
    n_cls = int(classes.max()) + 1
    cnt = torch.bincount(classes, minlength=n_cls)
    se = torch.bincount(classes, weights=errs, minlength=n_cls)
    overall = float(errs.mean().sqrt())
    if overall == 0.0:
        return 0.0
    ok = cnt >= CLASS_MIN
    if int(ok.sum()) < 2:
        return 0.0
    rms = (se[ok] / cnt[ok]).sqrt() / overall
    worst = float(rms.max())
    assert worst <= KAPPA, (tag, worst, int(torch.nonzero(ok).view(-1)[rms.argmax()]))
    return worst


def check_mlp(E, c, out, tag):
    sch = schedule(E, c)
    passes = [(0, "coarse", c.mc)] + ([(1, "fine", c.mf)] if c.nf else [])
    tol_max, tol_l2 = MLP_TOL[c.prec]
    worst = []
    ref_raw = {}
    for pas, key, m in passes:
        z = out[f"z_{key}"]
        ref = mlp64(c, params64(m), z)
        ref_raw[key] = ref
        got = out[f"raw_{key}"]
        assert bool(torch.isfinite(got).all()), (tag, key)
        for ch, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4))):
            em, el = errors(got[..., sl], ref[..., sl])
            print(f"{tag} MLP {key} {ch}: max {em:.2e}, L2 {el:.2e}")
            assert em <= tol_max and el <= tol_l2, (tag, key, ch, em, el)
    for ch, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4))):
        errs, cls = [], []
        for pas, key, _ in passes:
            d = out[f"raw_{key}"][..., sl].double() - ref_raw[key][..., sl]
            errs.append(d.pow(2).sum(-1).reshape(-1))
            cls.append(sample_classes(E, c, sch, pas))
        worst.append(check_uniformity(f"{tag} {ch}", torch.cat(errs), torch.cat(cls)))
    print(f"{tag} schedule uniformity: worst class RMS / overall RMS rgb {worst[0]:.2f}, sigma {worst[1]:.2f}")
    return ref_raw


def coarse_depths32(E, c):
    """The coarse depths by the FP32 formula, one torch op per operation (as the kernel rounds them)."""
    t = E.eng.linspace(c.nc).view(1, -1)
    z = (NEAR * (1.0 - t) + FAR * t).expand(c.n, c.nc)
    if c.perturb:
        mid = 0.5 * (z[:, 1:] + z[:, :-1])
        upper = torch.cat((mid, z[:, -1:]), dim=-1)
        lower = torch.cat((z[:, :1], mid), dim=-1)
        z = lower + (upper - lower) * c.noise["t_rand"]
    return z


def composite64(c, raw, z, noise):
    raw = f64(raw).clone()
    if c.bg is not None:
        raw[:, -1, :3] = f64(c.bg)
    return O.composite(raw, f64(z), f64(c.rd), c.noise_std, f64(noise), c.white, c.bg is not None)


def check_compositing(c, out, tag):
    refs = {}
    for key, sfx in (("coarse", "c"), ("fine", "f")):
        if key == "fine" and not c.nf:
            continue
        rgb, disp, acc, w, _ = composite64(c, out[f"raw_{key}"], out[f"z_{key}"], c.noise.get(f"n_{sfx}"))
        refs.update({f"rgb_{key}": rgb, f"disp_{key}": disp, f"acc_{key}": acc, "w_last": w[:, -1]})
        refs[f"w_{key}"] = w
    worst = 0.0
    for name in NAMES:
        if name not in refs:
            continue
        got, ref = out[name].reshape(refs[name].shape), refs[name]
        assert bool(torch.isfinite(got).all()), (tag, name)
        err = float((got.double() - ref).abs().max()) / max(1.0, float(ref.abs().max()))
        worst = max(worst, err)
        assert err <= COMP_TOL, (tag, name, err)
    print(f"{tag} compositing: worst {worst:.2e}")
    return refs


def resample_bounds(c, z_c, w, u, e):
    """Per-sample bounds [lower, upper] of the kernel's fine samples.  The kernel's FP32 cdf differs from the float64 cdf
    of the same weights by at most e per entry, and the inverse CDF is non-decreasing in u, so (where both take the same
    branch of the den < 1e-5 clamp) its sample at u lies between the float64 samples at u - e and u + e; that is the bound
    (cdf error / den) x bin width.  Where the float64 den lies within 2e of the clamp, either branch is accepted: the bound
    widens to the whole bin.  Sorting is monotone per element, so the sorted bounds bound the sorted samples."""
    bins = 0.5 * (z_c[:, 1:] + z_c[:, :-1])
    weights = w[:, 1:-1]
    nf = u.shape[1]
    lower = O.resample(bins, weights, nf, det=False, u=u - e)
    upper = O.resample(bins, weights, nf, det=False, u=u + e)
    wt = weights + 1e-5
    cdf = torch.cumsum(wt / wt.sum(-1, keepdim=True), dim=-1)
    cdf = torch.cat((torch.zeros_like(cdf[:, :1]), cdf), dim=-1).contiguous()
    nb = cdf.shape[1]
    amb = ((cdf[:, 1:] - cdf[:, :-1]) - 1e-5).abs() <= 2 * e                      # bin b: [cdf[b], cdf[b+1]]
    camb = torch.cat((torch.zeros_like(amb[:, :1], dtype=torch.int64), amb.long().cumsum(-1)), dim=-1)
    b_lo = (torch.searchsorted(cdf, (u - e).contiguous(), right=True) - 1).clamp(0, nb - 2)
    b_hi = (torch.searchsorted(cdf, (u + e).contiguous(), right=True) - 1).clamp(0, nb - 2)
    widen = (camb.gather(1, b_hi + 1) - camb.gather(1, b_lo)) > 0
    lower = torch.where(widen, torch.minimum(lower, bins.gather(1, b_lo)), lower)
    upper = torch.where(widen, torch.maximum(upper, bins.gather(1, b_hi + 1)), upper)
    return lower, upper, int(widen.sum())


def cdf_error_bound(nc, w):
    """FP32 cdf error per entry, per ray [n, 1].  The kernel's weights carry absolute errors of a few roundings each (one
    expf, 1 - alpha, a product of at most nc factors), which the normalisation divides by total = sum(w + 1e-5), small on
    transparent rays; the cdf sum (a per-lane run of at most 16 additions, a 5-level warp scan, 16 more) adds at most 40
    roundings of a quantity <= 1.  Bound: (nc + 40) roundings / min(total, 1)."""
    total = (w[:, 1:-1] + 1e-5).sum(-1, keepdim=True)
    return (nc + 40) * U32 / total.clamp(max=1.0)


def check_resampling(E, c, out, refs, tag):
    zc, zf = out["z_coarse"], out["z_fine"]
    n, S = zf.shape
    assert bool((zf[:, 1:] >= zf[:, :-1]).all()), (tag, "z_fine not sorted")
    # every coarse depth, bit for bit, as a multiset: coarse value k of a run of equal values matches the same offset in
    # z_fine's run
    first = torch.searchsorted(zf, zc.contiguous())
    off = torch.arange(c.nc, device=zc.device).view(1, -1) - torch.searchsorted(zc.contiguous(), zc.contiguous())
    idx = first + off
    assert bool((idx < S).all()), (tag, "a coarse depth is missing from z_fine")
    assert torch.equal(zf.gather(1, idx), zc), (tag, "a coarse depth is missing from z_fine")
    keep = torch.ones_like(zf, dtype=torch.bool)
    keep.scatter_(1, idx, False)
    rem = zf[keep].view(n, c.nf).double()
    u = c.noise["u"] if c.perturb else E.eng.linspace(c.nf).view(1, -1).expand(n, c.nf)
    e = cdf_error_bound(c.nc, refs["w_coarse"])
    lower, upper, n_amb = resample_bounds(c, f64(zc), refs["w_coarse"], f64(u), e)
    lo_s = torch.sort(lower, dim=-1).values - Z_SLACK
    hi_s = torch.sort(upper, dim=-1).values + Z_SLACK
    below, above = (lo_s - rem).clamp(min=0), (rem - hi_s).clamp(min=0)
    bad = int(((below > 0) | (above > 0)).sum())
    width = float((hi_s - lo_s).median())
    print(f"{tag} resampling: cdf error bound {float(e.min()):.1e}-{float(e.max()):.1e}, median bound width {width:.1e}, {n_amb} samples in ambiguous bins, "
          f"{bad} outside (by up to {max(float(below.max()), float(above.max())):.1e})")
    assert bad == 0, (tag, bad)


def check_stages(E, c, tag):
    out = render(E, c)
    # (a) coarse depths
    assert torch.equal(out["z_coarse"], coarse_depths32(E, c)), (tag, "z_coarse")
    # (b) MLP
    check_mlp(E, c, out, tag)
    # (c) compositing
    refs = check_compositing(c, out, tag)
    # (d) resampling and sort
    if c.nf:
        check_resampling(E, c, out, refs, tag)
    return out


# ---------------------------------------------------------------------------------------------------------------- stages
def _counts(nc, nf):
    return lambda E, prec: make_case(E, two_iter_rays(E), nc, nf, prec, seed=nc + nf)


def _opt(**kw):
    return lambda E, prec: make_case(E, two_iter_rays(E), 64, 64, prec, seed=7, **kw)


CASES = {
    # the 512^2 frame at 64c+128f in one launch, every ray, through in-kernel ray generation
    "frame512_64c128f": lambda E, prec: camera_case(E, 512, 0, 512, 64, 128, prec),
    # a 128-row band of the 1024^2 frame at 128c+256f: one ray per unit, many units per CTA
    "band1024_128c256f": lambda E, prec: camera_case(E, 1024, 448, 128, 128, 256, prec),
    # 4 * SMs + 37 rays at sample counts that fill, straddle and split tiles
    "64c64f": _counts(64, 64),
    "128c128f": _counts(128, 128),       # two rays per unit at exactly 256 samples: full tiles
    "129c128f": _counts(129, 128),       # one ray per unit from here: 1-row last tiles
    "100c60f": _counts(100, 60),         # rays straddle tiles and 8-row groups
    "200c300f": _counts(200, 300),
    "256c256f": _counts(256, 256),
    "40c24f": _counts(40, 24),
    "3c5f": _counts(3, 5),               # smallest fine resampling: 2 bins, 1 interior weight
    "32c1f": _counts(32, 1),
    "3c0f": _counts(3, 0),               # coarse only
    # options
    "perturb_noise": _opt(perturb=True, noise_std=0.1),
    "white_nobg": _opt(white=True, bg=False),
    "nobg": _opt(bg=False),
    "dir_z": _opt(dir_z=True),
    "perturb_100c60f": lambda E, prec: make_case(E, two_iter_rays(E), 100, 60, prec, perturb=True, noise_std=0.1, seed=9),
    # 1, 2 and 3 rays: a partly valid unit, idle CTAs
    "1ray": lambda E, prec: make_case(E, 1, 64, 128, prec, seed=1),
    "2rays": lambda E, prec: make_case(E, 2, 64, 128, prec, seed=2),
    "3rays": lambda E, prec: make_case(E, 3, 64, 128, prec, seed=3),
    # random-init weights: the transparent regime
    "random_init": lambda E, prec: make_case(E, two_iter_rays(E), 64, 128, prec, stress=False, seed=4),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(CASES))
def test_stages_against_float64(E, case, prec):
    c = CASES[case](E, prec)
    check_stages(E, c, f"{case} {prec}")


# ---------------------------------------------------------------------------------------------------------------- FP16 range
F16_INF = {"fast": 65520.0, "exact": 131024.0}  # smallest activation that the FP16 conversion (fast: one half; exact:
                                                # hi saturated at 65504 + lo) turns into inf
RANGE_MARGIN = {"fast": 1.02, "exact": 1.001}    # how far the kernel's FP32-accumulated activation can sit from float64
RANGE_TOL_EXACT_SAT = 1e-4                        # exact mode with activations in (65504, 131008)


def stored_weight(w, prec):
    """The FP32 value of the kernel's FP16 copy of a weight (fast: hi; exact: hi + lo), subnormals included."""
    hi = w.half()
    if prec == "fast":
        return hi.double()
    return hi.double() + (w - hi.float()).half().double()


def layer1_max(c, p, z):
    """float64 max |h1| (output of layers_xyz.1) per sample, and max |activation| per layer."""
    n, S = z.shape
    pts = (c.ro[:, None, :] + c.rd[:, None, :] * z[:, :, None]).reshape(-1, 3).double()
    dirs = dir_cols64(c)[torch.arange(n * S, device=z.device) // S]
    acts = O.mlp_activations(p, torch.cat((TR._posenc(pts, 10, True), TR._posenc(dirs, 4, False)), -1), f64(c.expr), f64(c.latent))
    return acts[1].abs().amax(-1).view(n, S), [float(a.abs().max()) for a in acts]


@pytest.mark.parametrize("prec", PRECS)
def test_fp16_range_of_hidden_activations(E, prec):
    """layers_xyz.1 (weight and bias) x g and layers_xyz.2's weight x 1/g leave the function unchanged and move the largest
    hidden activation to about 2^14 (within the normal tolerance), into (65504, 131008) (exact mode: correct; fast mode:
    non-finite) and beyond 131008 (non-finite in both).  A sample is never finite and wrong: every raw output either meets
    the tolerance or is non-finite, and so is every one of the seven outputs.  The reference uses layers_xyz.2's weight as
    the kernel stores it (FP16, deep in the subnormal range at these gains), so only the activations' range is tested."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=30)
    base = render(E, c)
    nets = {"coarse": c.mc, "fine": c.mf}
    amax = {}
    for key, m in nets.items():
        h1, per_layer = layer1_max(c, params64(m), base[f"z_{key}"])
        amax[key] = float(h1.max())
        print(f"{prec} {key}: max |activation| per layer (layers_xyz.0-5, layers_dir.0-2) {[f'{v:.3g}' for v in per_layer]}, "
              f"headroom to 65504: {65504.0 / max(per_layer):.3g}x")
    for target in (2.0 ** 14, 1.0e5, 4.5e5):
        # exact mode beyond 65504: hi saturates and lo carries the remainder with 11 bits, so those activations are only
        # FP16-accurate (relative 2^-12 of the part above 65504)
        tol_max = RANGE_TOL_EXACT_SAT if prec == "exact" and target > 65504.0 else MLP_TOL[prec][0]
        gains = {key: target / amax[key] for key in nets}
        models, refp = {}, {}
        for key, m in nets.items():
            g = gains[key]
            p = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
            p["layers_xyz.1.weight"] *= g
            p["layers_xyz.1.bias"] *= g
            p["layers_xyz.2.weight"] /= g
            models[key] = model(E, 0, True, params=p)
            w2 = dict(models[key].named_parameters())["layers_xyz.2.weight"].detach()
            refp[key] = params64(models[key], {"layers_xyz.2.weight": stored_weight(w2, prec)})
        c2 = types.SimpleNamespace(**vars(c))
        c2.mc, c2.mf = models["coarse"], models["fine"]
        out = render(E, c2)
        thr, mg = F16_INF[prec], RANGE_MARGIN[prec]
        n_over = n_nonfinite = 0
        worst = 0.0
        raw_ref = {}
        for key in nets:
            z = out[f"z_{key}"]
            zf = torch.where(torch.isfinite(z), z, base[f"z_{key}"])  # non-finite depths (after a non-finite coarse pass)
            ref = mlp64(c2, refp[key], zf)
            raw_ref[key] = ref
            act = layer1_max(c2, refp[key], zf)[0] if target > 2.0 ** 14 else None
            got = out[f"raw_{key}"].double()
            fin = torch.isfinite(got).all(-1) & torch.isfinite(z)
            scale = ref.abs().amax(dim=(0, 1))
            err = ((got - ref).abs() / scale).amax(-1)
            ok = fin & (err <= tol_max)
            assert bool((ok | ~fin).all()), (prec, target, key, "finite and wrong", float(err[fin].max()))
            worst = max(worst, float(err[fin].max()) if bool(fin.any()) else 0.0)
            if act is not None:
                over, under = act > thr * mg, act < thr / mg
                # (a fine sample of a ray whose coarse pass went non-finite has a non-finite depth)
                assert bool(fin[under & torch.isfinite(z)].all()), (prec, target, key, "non-finite below the FP16 limit")
                assert not bool(fin[over].any()), (prec, target, key, "finite beyond the FP16 limit")
                n_over += int(over.sum())
            else:
                assert bool(fin.all()), (prec, target, key, "non-finite at 2^14")
            n_nonfinite += int((~fin).sum())
        # the seven outputs: each within the tolerance of float64 compositing of the float64 raw, or non-finite
        n_bad_out = 0
        for key, sfx in (("coarse", "c"), ("fine", "f")):
            zf = torch.where(torch.isfinite(out[f"z_{key}"]), out[f"z_{key}"], base[f"z_{key}"])
            rgb, disp, acc, w, _ = composite64(c2, raw_ref[key], zf, c.noise.get(f"n_{sfx}"))
            for name, ref in ((f"rgb_{key}", rgb), (f"disp_{key}", disp), (f"acc_{key}", acc)):
                got = out[name].double().reshape(ref.shape)
                fin = torch.isfinite(got)
                tol = (4e-2 if name.startswith("disp") else 4e-3) if prec == "fast" else 2e-4
                bad = fin & ((got - ref).abs() > tol * ref.abs().clamp(min=1.0))
                n_bad_out += int(bad.sum())
        print(f"{prec} max activation -> {target:.3g}: gains {gains['coarse']:.3g} / {gains['fine']:.3g}, {n_over} samples "
              f"beyond the FP16 limit, {n_nonfinite} non-finite raw samples, worst finite error {worst:.2e}")
        assert n_bad_out == 0, (prec, target, n_bad_out)
        if target == 1.0e5 and prec == "exact":
            assert n_nonfinite == 0
        if target > 1.0e5 or prec == "fast" and target == 1.0e5:
            assert n_over > 0 and n_nonfinite > 0


# ---------------------------------------------------------------------------------------------------------------- non-finite
def reference_outputs_cpu(c, rays, pc, pf, bg, noise, expr):
    """float64 torch outputs (nerface_oracle.render_chunk) of the given rays, on the CPU."""
    cpu = lambda t: None if t is None else t.detach().double().cpu()  # noqa: E731
    n = rays.shape[0]
    r = torch.cat((cpu(rays[:, :3]), cpu(rays[:, 3:6]), torch.full((n, 1), NEAR, dtype=torch.float64),
                   torch.full((n, 1), FAR, dtype=torch.float64)), -1)
    with torch.no_grad():
        return O.render_chunk(r, {k: cpu(v) for k, v in pc.items()}, {k: cpu(v) for k, v in pf.items()},
                              O.Sampling(c.nc, c.nf, False, c.noise_std, c.white, 65536), cpu(expr), cpu(c.latent), cpu(bg),
                              O.Noise(n_c=cpu(noise.get("n_c")), n_f=cpu(noise.get("n_f"))))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("field", ["origin", "background", "sigma_noise", "weight", "expression"])
def test_nonfinite_inputs_give_nonfinite_outputs(E, field, bad, prec):
    """A NaN or +inf in one ray's origin, background or sigma-noise draw, in one entry of layers_xyz.1.weight, or in the
    expression: every output float64 torch makes non-finite is non-finite in the kernel's result too (never a finite
    value), and for the per-ray inputs every other ray is unchanged bit for bit."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, noise_std=0.1, seed=40)
    clean = render(E, c)
    ray = c.n // 2 + 1
    v = float(bad)
    pc, pf = params64(c.mc), params64(c.mf)
    expr = c.expr
    d = types.SimpleNamespace(**vars(c))
    if field == "origin":
        d.ro = c.ro.clone()
        d.ro[ray, 0] = v
    elif field == "background":
        d.bg = c.bg.clone()
        d.bg[ray, 1] = v
    elif field == "sigma_noise":
        d.noise = dict(c.noise)
        d.noise["n_c"] = c.noise["n_c"].clone()
        d.noise["n_c"][ray, c.nc // 2] = v
    elif field == "weight":
        p = {k: t.detach().cpu().clone() for k, t in c.mc.state_dict().items()}
        p["layers_xyz.1.weight"][17, 5] = v
        d.mc = model(E, 0, True, params=p)
        pc = params64(d.mc)
    else:
        expr = c.expr.clone()
        expr[3] = v
        d.expr = expr
    got = render(E, d)
    per_ray = field in ("origin", "background", "sigma_noise")
    rays = [ray] if per_ray else [0, c.n // 3, c.n - 1]
    sel = torch.tensor(rays, device=E.dev)
    ref = reference_outputs_cpu(d, torch.cat((d.ro, d.rd), -1)[sel], pc, pf, d.bg[sel],
                                {k: t[sel] for k, t in d.noise.items()}, expr)
    reached = 0
    for name, r in zip(NAMES, ref):
        g = got[name][sel].cpu().reshape(r.shape)
        nonfin = ~torch.isfinite(r)
        reached += int(nonfin.sum())
        assert bool((~torch.isfinite(g[nonfin])).all()), (field, bad, name, "finite where torch gives a non-finite value")
        if not per_ray and bool(nonfin.all()):  # the network or the frame: every ray is affected alike
            assert not bool(torch.isfinite(got[name]).any()), (field, bad, name, "finite where torch gives a non-finite value")
    if per_ray:
        others = torch.ones(c.n, dtype=torch.bool, device=E.dev)
        others[ray] = False
        for name in NAMES:
            assert torch.equal(got[name][others], clean[name][others]), (field, bad, name, "another ray changed")
    print(f"{field} = {bad} ({prec}): {reached} output entries non-finite in float64 torch, all non-finite in the kernel")
