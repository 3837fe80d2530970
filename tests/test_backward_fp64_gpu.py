"""The fused backward (csrc/nfb_train.cu) against a float64 reference of the same gradients, at the production batch, at the
persistent kernels' scheduling boundaries, at sample counts that fill tiles partly or straddle rays across tiles, with every
compositing option, at the edges of the power-of-two loss scale and through the over-budget chunked path.

The reference is tests/torch_reference.render_at_depths evaluated in float64 on the GPU at the depths the kernel sampled
(pinned to the reference's own autograd by test_backward_reference_cpu.py).  Parameter gradients are linear in the per-ray
output gradients, so it runs in ray chunks and adds the gradients up.

Every case compares all 48 used parameter gradients and the latent gradient, per tensor:
  max |got - ref| <= tol_max * max |ref|        (as in test_backward_gpu.py)
  |got - ref|_2   <= tol_l2  * |ref|_2          (catches errors spread over many entries that stay under the max bound)
The backward carries FP16 operands in both precision modes; in fast mode the forward's saved state (colours, sigma inputs,
activations) carries FP16 rounding as well.  Measured on an H100 80GB HBM3 (CUDA 12.9), worst tensor over all cases:
  dense, exact        max 1.7e-3, L2 7.2e-4                 -> TOL exact  (5e-3, 2e-3)
  dense, fast         max 1.8e-2, L2 1.2e-2                 -> TOL fast   (4e-2, 3e-2)
  3c+0f, fast         max 6.4e-2, L2 4.2e-2 (intervals of 0.3: d alpha / d sigma = delta exp(-sigma delta) turns the fast
                      forward's sigma rounding into percent-level changes)   -> (1.5e-1, 1e-1)
  single ray, exact   max 1.8e-2, L2 5.6e-3                 -> PROBE_TOL exact (5e-2, 2e-2)
  single ray, fast    max 1.6e-1, L2 1.0e-1                 -> PROBE_TOL fast  (4e-1, 3e-1); a dropped or doubled tile
                      moves a probe ray's gradient by 100 %
  d raw per pass      L2 8.3e-4 (exact) / 4.9e-2 (fast)     -> DRAW_L2 3e-3 / 1e-1
  forward outputs     max abs 1.5e-5 (exact) / 2.3e-3 (fast) -> FWD_TOL 5e-5 / 1e-2
"""
import ctypes as C
import types

import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_gpu import decode_image, dev_tensor, dy_off

pytestmark = pytest.mark.gpu

NEAR, FAR = 0.2, 0.8
NAMES = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
TOL = {"exact": (5e-3, 2e-3), "fast": (4e-2, 3e-2)}      # (max, L2) of dense parameter gradients
TOL_3C_FAST = (1.5e-1, 1e-1)
PROBE_TOL = {"exact": (5e-2, 2e-2), "fast": (4e-1, 3e-1)}  # single-ray gradients
DRAW_L2 = {"exact": 3e-3, "fast": 1e-1}                    # d raw, relative L2 per pass
ACC_NOISE = 5e-6  # acc-only gradients / rgb-only gradients: measured 5.6e-7 (kernel), 4.4e-7 (float64)
FWD_TOL = {"exact": 5e-5, "fast": 1e-2}                    # forward outputs, absolute
PRECS = ["exact", "fast"]


@pytest.fixture(scope="module")
def E(built_lib):
    import nerf
    from nerf import _capi, _engine
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    e = types.SimpleNamespace(nerf=nerf, capi=_capi, dev=torch.device("cuda", 0))
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
    """4 * SMs + 37 rays: at two rays per unit that is 2 * SMs + 19 units, so every CTA of the persistent chain and render
    kernels runs at least two units (ring parity across tiles, operand-buffer reuse, the barrier between tiles) and the
    last unit is half filled."""
    return 4 * E.sms + 37


def make_case(E, n, nc, nf, prec, stress=True, perturb=True, noise_std=0.1, bg=True, white=False, dir_z=False, seed=0):
    g = torch.Generator().manual_seed(1000 + seed)
    nz = O.draw_noise(n, O.Sampling(nc, nf, perturb, noise_std, white, 2048), g)
    noise = {k: getattr(nz, k).to(E.dev) for k in ("t_rand", "n_c", "u", "n_f") if getattr(nz, k) is not None}
    return types.SimpleNamespace(
        n=n, nc=nc, nf=nf, prec=prec, perturb=perturb, noise_std=noise_std, white=white, noise=noise,
        ro=E.ro[:n].contiguous(), rd=E.rd[:n].contiguous(), bg=E.bg[:n].contiguous() if bg else None,
        dz=(torch.rand(n, generator=g) * 2.0 - 1.0).to(E.dev) if dir_z else None, expr=E.expr, latent=E.latent,
        mc=model(E, 100, stress), mf=model(E, 101, stress) if nf > 0 else None)


def train_forward(E, c):
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    return E.eng.render(c.ro, c.rd, NEAR, FAR, c.nc, c.nf, perturb=c.perturb, noise_std=c.noise_std, white_bkgd=c.white,
                        background=c.bg, dir_z=c.dz, noise=c.noise, precision=c.prec, train=True)


def saved_state(E, c):
    """Sample depths, d raw and the loss scale of the last (one-launch) training forward / backward."""
    torch.cuda.synchronize()
    d = E.eng.train_debug()
    s = types.SimpleNamespace(dbg=d, R=d.rays_per_unit, tc=d.tiles_coarse, tf=d.tiles_fine, n_tiles=int(d.n_tiles))
    s.z_c = dev_tensor(d.z_coarse, (c.n, c.nc)).clone()
    s.z_f = dev_tensor(d.z_fine, (c.n, c.nc + c.nf)).clone() if c.nf else None
    return s


def kernel_backward(E, c, gouts):
    pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
    pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER] if c.mf is not None else None
    gc, gf, gl = E.eng.backward(list(gouts), pc, pf)
    torch.cuda.synchronize()
    return gc, gf, gl


def reference(E, c, z_c, z_f, gouts, lo=0, hi=None, want_draw=False, want_taps=None):
    """float64 outputs, parameter / latent gradients of sum_i <out_i, gouts_i> over rays [lo, hi); with want_draw also
    dL/d raw per pass, with want_taps = "a<L>" the gradient of layer L's pre-activation (both passes, every chunk)."""
    hi = c.n if hi is None else hi
    f64 = lambda t: None if t is None else t.detach().to(E.dev, torch.float64)  # noqa: E731
    pc = {k: f64(v).requires_grad_(True) for k, v in c.mc.named_parameters()}
    pf = {k: f64(v).requires_grad_(True) for k, v in c.mf.named_parameters()} if c.mf is not None else None
    lat, expr = f64(c.latent).requires_grad_(True), f64(c.expr)
    rays = torch.cat((c.ro, c.rd, torch.full((c.n, 1), NEAR, device=E.dev), torch.full((c.n, 1), FAR, device=E.dev)), -1).double()
    chunk = max(16, 65536 // (2 * c.nc + c.nf))
    outs, draw, tapped = [[] for _ in NAMES], {"coarse": [], "fine": []}, []
    for b in range(lo, hi, chunk):
        s = slice(b, min(hi, b + chunk))
        taps = {} if want_draw or want_taps else None
        o = TR.render_at_depths(rays[s], pc, pf, expr, lat, f64(z_c[s]), f64(z_f[s]) if z_f is not None else None, NEAR, FAR,
                                c.noise_std, {k: f64(v[s]) for k, v in c.noise.items()}, c.white,
                                f64(c.bg[s]) if c.bg is not None else None, f64(c.dz[s]) if c.dz is not None else None, taps)
        loss = sum(((oi * f64(gi[s])).sum() for oi, gi in zip(o, gouts) if oi is not None and gi is not None),
                   torch.zeros((), dtype=torch.float64, device=E.dev))
        loss.backward()
        for i, oi in enumerate(o):
            if oi is not None:
                outs[i].append(oi.detach())
        for key, t in (taps or {}).items():
            if want_draw:
                draw[key].append(t["raw"].grad)
            if want_taps:
                tapped.append(t[want_taps].grad)
    return types.SimpleNamespace(outs=[torch.cat(x) if x else None for x in outs], gc=[pc[k].grad for k in TR.PARAM_ORDER],
                                 gf=[pf[k].grad for k in TR.PARAM_ORDER] if pf is not None else None, glat=lat.grad,
                                 draw={k: torch.cat(v) for k, v in draw.items() if v}, taps=tapped)


def flat(kg):
    """The kernel's gradient tensors of one backward call (both networks, the latent) as one list."""
    return [t for t in list(kg[0]) + list(kg[1] or []) + [kg[2]] if t is not None]


def grad_pairs(kg, R):
    gc, gf, gl = kg
    out = []
    for net, gs, rs in (("coarse", gc, R.gc), ("fine", gf, R.gf)):
        if rs is None:
            assert gs is None
            continue
        for k, g, r in zip(TR.PARAM_ORDER, gs, rs):
            if k.startswith("layers_dir.3"):  # unused by the forward: no gradient on either side
                assert g is None and r is None
                continue
            out.append((f"{net}/{k}", g, r))
    out.append(("latent", gl, R.glat))
    return out


def errors(got, ref):
    """(max-abs error / max |ref|, relative L2 error); a reference that is exactly zero must be met exactly."""
    got, ref = got.double(), ref.double()
    rmax = float(ref.abs().max())
    if rmax == 0.0:
        return (0.0, 0.0) if float(got.abs().max()) == 0.0 else (float("inf"), float("inf"))
    return float((got - ref).abs().max()) / rmax, float((got - ref).norm() / ref.norm())


def check(tag, pairs, tol, quiet=False):
    tol_max, tol_l2 = tol
    worst = [0.0, 0.0, "", ""]
    for name, g, r in pairs:
        assert g is not None and r is not None, (tag, name)
        assert bool(torch.isfinite(g).all()), (tag, name, "non-finite kernel gradient")
        em, el = errors(g, r)
        if em >= worst[0]:
            worst[0], worst[2] = em, name
        if el >= worst[1]:
            worst[1], worst[3] = el, name
    if not quiet:
        print(f"{tag}: worst max {worst[0]:.2e} ({worst[2]}), worst L2 {worst[1]:.2e} ({worst[3]})")
    assert worst[0] <= tol_max and worst[1] <= tol_l2, (tag, worst)
    return worst[0], worst[1]


def rowmap(c, s, pas):
    """(tile, row) of every (ray, sample) of one pass in the records / d raw."""
    Sx = c.nc + c.nf if pas else c.nc
    gi = torch.arange(c.n).view(-1, 1).expand(c.n, Sx)
    ii = torch.arange(Sx).view(1, -1).expand(c.n, Sx)
    unit, rr = gi // s.R, gi % s.R
    prow = rr * Sx + ii
    tile = unit * (s.tc + s.tf) + (s.tc if pas else 0) + prow // 128
    return tile.reshape(-1).to(c.ro.device), (prow % 128).reshape(-1).to(c.ro.device)


def check_draw(tag, c, s, R):
    """d raw per pass against dL/d raw of the reference (relative L2; the max-abs error is printed only: a sigma input
    within the forward's rounding of zero flips its ReLU, which moves single entries by their own size); rows that belong
    to no sample stay zero."""
    d_raw = dev_tensor(s.dbg.d_raw, (s.n_tiles, 128, 4))
    used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=d_raw.device)
    for pas, key in ((0, "coarse"), (1, "fine")):
        if key not in R.draw:
            continue
        tile, row = rowmap(c, s, pas)
        used[tile, row] = True
        em, el = errors(d_raw[tile, row], R.draw[key].reshape(-1, 4))
        print(f"{tag} d raw {key}: max {em:.2e}, L2 {el:.2e}")
        assert el <= DRAW_L2[c.prec], (tag, key, em, el)
    if bool((~used).any()):
        assert float(d_raw[~used].abs().max()) == 0.0


def out_grads(E, c, seed=5, which=None):
    """A loss with nonzero, ray-varying gradients on all seven outputs (or only on `which`)."""
    g = torch.Generator().manual_seed(seed)
    n = c.n
    shapes = [(n, 3), (n,), (n,), (n, 3), (n,), (n,), (n,)]
    go = [((torch.rand(sh, generator=g) - 0.3) / n).to(E.dev) for sh in shapes]
    if c.nf == 0:
        go[3] = go[4] = go[5] = None
    if which is not None:
        go = [t if i == which else (None if t is None else torch.zeros_like(t)) for i, t in enumerate(go)]
    return go


def full_case(E, c, tag, gouts=None, draw=True, tol=None):
    out = train_forward(E, c)
    s = saved_state(E, c)
    gouts = out_grads(E, c) if gouts is None else gouts
    kg = kernel_backward(E, c, gouts)
    R = reference(E, c, s.z_c, s.z_f, gouts, want_draw=draw)
    fwd = max(float((out[nme].double() - R.outs[i]).abs().max()) for i, nme in enumerate(NAMES) if R.outs[i] is not None)
    print(f"{tag} forward: max abs {fwd:.2e}")
    assert fwd <= FWD_TOL[c.prec], tag
    if draw:
        check_draw(tag, c, s, R)
    return out, s, kg, R, check(tag, grad_pairs(kg, R), tol or TOL[c.prec])


# ---------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("prec", PRECS)
def test_production_batch_dense(E, prec):
    """2048 rays at 64c+64f (1024 units, 3072 tiles: every chain CTA runs 7-8 units, every weight-gradient CTA sums ~190
    tiles), perturbation, sigma noise and a background, random-init weights (the start of training), called as the fused
    trainer calls the library: training forward, nfb_loss_mse_grad, backward; plus terms on the other five outputs."""
    c = make_case(E, 2048, 64, 64, prec, stress=False)
    out = train_forward(E, c)
    s = saved_state(E, c)
    n = c.n
    g = torch.Generator().manual_seed(11)
    target = torch.rand(n, 3, generator=g).to(E.dev)
    grad_c, grad_f = torch.zeros(n, 3, device=E.dev), torch.zeros(n, 3, device=E.dev)
    loss = torch.zeros(2, device=E.dev)
    E.eng.loss_mse_grad(out["rgb_coarse"], out["rgb_fine"], target, n, grad_c, grad_f, loss)
    torch.cuda.synchronize()
    for rgb, gr in ((out["rgb_coarse"], grad_c), (out["rgb_fine"], grad_f)):
        ref = 2.0 * (rgb.double() - target.double()) / (3 * n)
        assert float((gr.double() - ref).abs().max()) <= 1e-6 * float(ref.abs().max())
    w = lambda scale: (torch.rand(n, generator=g) * scale / n).to(E.dev)  # noqa: E731
    gouts = [grad_c, w(0.3), w(0.2), grad_f, w(0.1), w(0.2), w(0.5)]
    kg = kernel_backward(E, c, gouts)
    R = reference(E, c, s.z_c, s.z_f, gouts, want_draw=True)
    for i, nme in enumerate(NAMES):
        err = float((out[nme].double() - R.outs[i]).abs().max())
        print(f"{prec} forward {nme}: max abs {err:.2e}")
        assert err <= FWD_TOL[prec], nme
    check_draw(f"dense {prec}", c, s, R)
    check(f"dense 2048r {prec}", grad_pairs(kg, R), TOL[prec])


# ---------------------------------------------------------------------------------------------------------------- (b)
def probe_units(E, n_units, tc, tf):
    """Units at the scheduling boundaries: the chain / render CTAs' first and second iterations (CTA b runs units b, b+grid,
    ...) and the last unit; for the weight-gradient kernel the tiles either side of every CTA's share boundary."""
    grid = min(n_units, E.sms)
    units = {0, grid - 1, grid, 2 * grid - 1, n_units - 1}
    buf = (C.c_uint32 * 16)(E.sms, n_units * tc, n_units * tf)
    assert E.capi.lib.nfb_debug_schedule(4, 0, buf, 16) == 3
    for t_cnt, parts in ((tc, int(buf[0])), (tf, int(buf[1]))):
        if parts == 0:
            continue
        total = n_units * t_cnt
        per = (total + parts - 1) // parts
        for k in range(parts + 1):
            for tile in (k * per - 1, k * per):
                if 0 <= tile < total:
                    units.add(tile // t_cnt)
    return sorted(u for u in units if 0 <= u < n_units)


@pytest.mark.parametrize("prec", PRECS)
def test_scheduling_boundary_probes(E, prec):
    """2047 rays (the last unit half filled), one training forward, then one backward per probe ray with output gradients
    on that ray only, each against the float64 gradient of that single ray.  A tile the chain or weight-gradient kernel drops,
    doubles or misroutes at a CTA boundary shows up here as a zero or wrong single-ray gradient.  Also pins that the backward
    can be repeated on one saved forward (each call zeroes d raw, the scale and the accumulators)."""
    c = make_case(E, 2047, 64, 64, prec, seed=2)
    train_forward(E, c)
    s = saved_state(E, c)
    n_units = (c.n + s.R - 1) // s.R
    units = probe_units(E, n_units, s.tc, s.tf)
    rays = [u * s.R + r for u in units for r in range(s.R) if u * s.R + r < c.n]
    assert (n_units - 1) * s.R + 1 == c.n and c.n - 1 in rays  # the half-filled last unit is probed
    dense = out_grads(E, c, seed=3)
    worst = [0.0, 0.0]
    first = None
    for i in rays:
        gouts = []
        for t in dense:
            z = torch.zeros_like(t)
            z[i] = t[i] * c.n
            gouts.append(z)
        kg = kernel_backward(E, c, gouts)
        if first is None:  # the same output gradients again: the same gradients up to the order of the atomics
            again = kernel_backward(E, c, gouts)
            rep = max(float((a - b).abs().max()) / float(a.abs().max()) for a, b in zip(flat(kg), flat(again)))
            print(f"{prec}: repeated backward, worst relative difference {rep:.2e}")
            assert rep <= 1e-6
            first = i
        R = reference(E, c, s.z_c, s.z_f, gouts, lo=i, hi=i + 1)
        em, el = check(f"probe ray {i} (unit {i // s.R})", grad_pairs(kg, R), PROBE_TOL[prec], quiet=True)
        worst = [max(worst[0], em), max(worst[1], el)]
    print(f"{prec}: {len(rays)} probe rays in units {units}; worst max {worst[0]:.2e}, worst L2 {worst[1]:.2e}")


# ---------------------------------------------------------------------------------------------------------------- (c)
SHAPES = [(64, 64), (64, 128), (100, 60), (40, 24), (256, 256), (64, 0), (3, 0)]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("nc,nf", SHAPES, ids=[f"{a}c{b}f" for a, b in SHAPES])
def test_shapes(E, nc, nf, prec):
    """two_iter_rays rays.  Sample counts that fill tiles partly (40+24, 3+0), straddle rays across tiles (100+60), use one ray per unit at the
    512-sample limit (256+256: 16 samples per lane in the compositing backward), and coarse-only networks (no fine model)."""
    c = make_case(E, two_iter_rays(E), nc, nf, prec, seed=nc + nf)
    full_case(E, c, f"{nc}c{nf}f {prec}", tol=TOL_3C_FAST if (nc, prec) == (3, "fast") else None)


# ---------------------------------------------------------------------------------------------------------------- (d)
OPTIONS = {"white_nobg": dict(white=True, bg=False), "nobg": dict(bg=False), "dir_z": dict(dir_z=True),
           "deterministic": dict(perturb=False, noise_std=0.0)}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("nc,nf", [(64, 64), (100, 60)], ids=["64c64f", "100c60f"])
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_compositing_options(E, opt, nc, nf, prec):
    c = make_case(E, two_iter_rays(E), nc, nf, prec, seed=7, **OPTIONS[opt])
    full_case(E, c, f"{opt} {nc}c{nf}f {prec}")


@pytest.mark.parametrize("prec", PRECS)
def test_each_output_gradient_alone(E, prec):
    """One backward per output (rgb, disp, acc of each pass, w_last) on one saved forward, on a white background without
    a background image, so every term of the compositing backward is checked on its own."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=8, white=True, bg=False)
    out = train_forward(E, c)
    s = saved_state(E, c)
    rgb_scale = {}
    for which, nme in enumerate(NAMES):
        gouts = out_grads(E, c, seed=9, which=which)
        kg = kernel_backward(E, c, gouts)
        R = reference(E, c, s.z_c, s.z_f, gouts, want_draw=True)
        pairs = grad_pairs(kg, R)
        if nme.startswith("rgb"):
            rgb_scale[nme[4:]] = {name: float(r.abs().max()) for name, _, r in pairs}
        if nme.startswith("acc"):
            # acc = 1 - prod(1 - alpha + 1e-10) is 1 to within rounding on every ray (the last interval is 1e10 long), so its
            # float64 gradient is below 1e-6 of the others and the kernel's is rounding noise of the reverse recurrence on the
            # same scale: bound it by the gradient the same-sized rgb output gradient of the same pass makes
            scale = rgb_scale[nme[4:]]
            noise = max(float(g.abs().max()) / scale[name] for name, g, _ in pairs if name in scale and scale[name] > 0)
            ref = max(float(r.abs().max()) / scale[name] for name, _, r in pairs if name in scale and scale[name] > 0)
            print(f"only {nme} {prec}: max |gradient| / rgb-gradient scale: kernel {noise:.2e}, float64 {ref:.2e}")
            assert all(bool(torch.isfinite(g).all()) for _, g, _ in pairs) and noise <= ACC_NOISE, (nme, noise)
            continue
        check_draw(f"only {nme} {prec}", c, s, R)
        check(f"only {nme} {prec}", pairs, TOL[prec])


# ---------------------------------------------------------------------------------------------------------------- (e)
@pytest.mark.parametrize("prec", PRECS)
def test_loss_scale_edges(E, prec):
    """The power-of-two loss scale: output gradients scaled by 2^k give gradients scaled by 2^k (up to the order of the
    atomics) while the scale stays inside scale_kernel's +-100 clamp; all-zero output gradients give exact zeros; output
    gradients spanning 1e4 across rays still meet the float64 tolerance."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=12)
    train_forward(E, c)
    s = saved_state(E, c)
    base = out_grads(E, c, seed=13)
    g0 = kernel_backward(E, c, base)
    worst = 0.0
    for k in (-60, -20, 20, 60):
        gk = kernel_backward(E, c, [t * 2.0 ** k for t in base])
        e = float(torch.log2(dev_tensor(s.dbg.scale, (2,))[0].double()))
        assert -100 < e < 100 and e == round(e), (k, e)
        for a, b in zip(flat(g0), flat(gk)):
            worst = max(worst, float((a.double() * 2.0 ** k - b.double()).abs().max() / b.double().abs().max()))
    print(f"{prec}: output gradients x 2^k, k = +-20, +-60: worst relative difference {worst:.2e}")
    assert worst <= 4e-6  # measured 8.7e-7 (exact) / 1.3e-6 (fast): the order of the weight-gradient atomics
    zero = kernel_backward(E, c, [torch.zeros_like(t) for t in base])
    assert all(float(t.abs().max()) == 0.0 and bool(torch.isfinite(t).all()) for t in flat(zero))
    g = torch.Generator().manual_seed(14)
    span = (10.0 ** (torch.rand(c.n, generator=g) * 4.0 - 2.0)).to(E.dev)
    gouts = [t * (span.view(-1, 1) if t.dim() == 2 else span) for t in base]
    kg = kernel_backward(E, c, gouts)
    check(f"1e4 span {prec}", grad_pairs(kg, reference(E, c, s.z_c, s.z_f, gouts)), TOL[prec])


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("field", [0, 3], ids=["rgb_coarse", "rgb_fine"])
def test_nonfinite_output_gradient_gives_nonfinite_gradients(E, bad, field, prec):
    """A NaN or +inf in one ray's output gradient: every parameter gradient the float64 reference (torch autograd) makes
    non-finite is non-finite in the kernel's result too, never a finite value.  (An inf reaches d raw together with NaN from
    inf - inf in the reverse recurrence; the chain's FP16 conversions keep inf rather than clamping it to 65504.)"""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=15)
    train_forward(E, c)
    s = saved_state(E, c)
    gouts = out_grads(E, c, seed=16)
    ray = c.n // 2
    gouts[field] = gouts[field].clone()
    gouts[field][ray, 1] = float(bad)
    kg = kernel_backward(E, c, gouts)
    R = reference(E, c, s.z_c, s.z_f, gouts, lo=ray, hi=ray + 1)
    reached = 0
    for name, g, r in grad_pairs(kg, R):
        if not bool(torch.isfinite(r).all()):
            reached += 1
            assert not bool(torch.isfinite(g).all()), (name, "finite gradient where torch gives a non-finite one")
    assert reached >= 24, reached  # every used parameter of the network that renders that output


# ---------------------------------------------------------------------------------------------------------------- (f)
def dy_images(s, c):
    """Largest |dY| per layer as stored in the tile records (FP16, loss-scaled), over both passes."""
    recs = dev_tensor(s.dbg.records, (s.n_tiles, s.dbg.record_bytes // 2), "<i2")
    out = []
    for layer in range(9):
        m = 0.0
        for pas in (0, 1):
            tile, row = rowmap(c, s, pas)
            img = decode_image(recs, dy_off(layer), 256 if layer < 6 else 128)[tile, row]
            m = max(m, float(img.abs().max()))
        out.append(m)
    return out


@pytest.mark.parametrize("prec", PRECS)
def test_chain_dynamic_range(E, prec):
    """The chain carries loss-scaled gradients in FP16.  At the stress weights no dY entry saturates (printed: the headroom,
    largest |dY| over all layers / max |d raw|).  Then the weights are re-balanced so that the forward is unchanged but
    dY of layers_xyz.4 grows by a factor chosen from the float64 taps to exceed FP16's 65504 after the loss scale
    (layers_xyz.4 divided by g, layers_xyz.5's weight multiplied by g): the kernel must return gradients within tolerance
    or non-finite ones, never finite, wrong, saturated ones."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=17)
    gouts = out_grads(E, c, seed=18)
    train_forward(E, c)
    s = saved_state(E, c)
    kernel_backward(E, c, gouts)
    scale = float(dev_tensor(s.dbg.scale, (2,))[0])
    d_raw = dev_tensor(s.dbg.d_raw, (s.n_tiles, 128, 4))
    dy = dy_images(s, c)
    assert max(dy) < 65504.0, dy
    head = max(dy) / (float(d_raw.abs().max()) * scale)
    print(f"{prec}: loss scale 2^{int(torch.log2(torch.tensor(scale)))}, max |dY| per layer (scaled) "
          f"{[f'{v:.3g}' for v in dy]}, headroom max|dY| / max|d raw| = {head:.3g}")

    # the gain that takes max |dY4| * scale to 4 x 65504, from the float64 dY4 (both passes)
    taps_max = max(float(t.abs().max()) for t in reference(E, c, s.z_c, s.z_f, gouts, want_taps="a4").taps)
    gain = 4.0 * 65504.0 / (taps_max * scale)
    assert gain > 1.0

    def rebalance(m):
        p = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
        p["layers_xyz.4.weight"] /= gain
        p["layers_xyz.4.bias"] /= gain
        p["layers_xyz.5.weight"] *= gain
        return model(E, 0, False, params=p)
    c.mc, c.mf = rebalance(c.mc), rebalance(c.mf)
    train_forward(E, c)
    s = saved_state(E, c)
    kg = kernel_backward(E, c, gouts)
    recs = dev_tensor(s.dbg.records, (s.n_tiles, s.dbg.record_bytes // 2), "<i2")
    dy4 = torch.cat([decode_image(recs, dy_off(4), 256)[rowmap(c, s, pas)] for pas in (0, 1)])
    pairs = grad_pairs(kg, reference(E, c, s.z_c, s.z_f, gouts))
    finite = all(bool(torch.isfinite(g).all()) for _, g, _ in pairs)
    print(f"{prec}: gain {gain:.3g} on dY4: {int((dy4.abs() == 65504.0).sum())} entries at 65504, "
          f"{int(torch.isinf(dy4).sum())} at inf -> kernel gradients {'finite' if finite else 'non-finite'}")
    if finite:
        check(f"rebalanced x{gain:.3g} {prec}", pairs, TOL[prec])


# ---------------------------------------------------------------------------------------------------------------- (g)
def chunked_case(E, prec):
    return make_case(E, two_iter_rays(E), 64, 64, prec, seed=19, dir_z=True)


@pytest.mark.parametrize("prec", PRECS)
def test_chunked_backward_against_float64(E, prec, monkeypatch):
    """Over the memory budget (48 MiB: 16 units of 3 one-MiB tiles = 32 rays per chunk, the last chunk ragged) the backward re-runs the training forward per chunk with every per-ray pointer advanced: rays, background, dir_z, the
    perturbation and sigma-noise draws.  Depths come from a one-launch forward of the same rays and noise."""
    c = chunked_case(E, prec)
    assert c.n % 32 != 0
    train_forward(E, c)
    s = saved_state(E, c)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    l0 = E.eng.launch_count()
    train_forward(E, c)
    gouts = out_grads(E, c, seed=20)
    kg = kernel_backward(E, c, gouts)
    assert E.eng.launch_count() - l0 > 5 * (c.n // 32)  # a SAVE forward and four backward launches per chunk
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    check(f"chunked {prec}", grad_pairs(kg, reference(E, c, s.z_c, s.z_f, gouts)), TOL[prec])


@pytest.mark.parametrize("tables", ["caller", "library"])
def test_chunked_backward_ignores_a_render_in_between(E, tables, monkeypatch):
    """Chunked training forward of frame A, a no_grad render of frame B (other expression, latent and sample counts), then
    the backward: the re-run forwards still differentiate frame A (its folded biases and, with the library's own linspace
    tables, its depth tables are saved with the training state).  Must equal the run without the render in between."""
    c = chunked_case(E, "fast")
    if tables == "library":  # NfbSampling.t_coarse / u_fine NULL: the handle's cached tables, which a new sample count replaces
        monkeypatch.setattr(E.eng, "linspace", lambda n: types.SimpleNamespace(data_ptr=lambda: None))
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    gouts = out_grads(E, c, seed=21)
    grads = []
    for interleave in (False, True):
        train_forward(E, c)
        if interleave:
            E.eng.set_frame(c.expr * 0.5 + 0.3, c.latent * -2.0 + 0.05)
            b = E.eng.render(c.ro[:100], c.rd[:100], NEAR, FAR, 96, 80, background=c.bg[:100], precision="fast")
            torch.cuda.synchronize()
            assert bool(torch.isfinite(b["rgb_fine"]).all())
        grads.append(flat(kernel_backward(E, c, gouts)))
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    for a, b in zip(*grads):
        assert float((a - b).abs().max()) <= 1e-6 * float(a.abs().max())
