"""The training forward (render_kernel<*, true>, csrc/nfb_render.cu) against float64 and against the evaluation forward, at
every tile of its persistent schedule, and at its FP16-range, empty-row and non-finite edges.

The training forward writes what the whole backward trusts: per 128-row tile the FP16 positional-encoding and
direction-encoding images, nine activation images and their ReLU masks, and per sample the colour and the ReLU input of
sigma.  Each case runs the training forward (eng.render(train=True), read through eng.train_debug()) and the evaluation
forward (debug=True) on the same inputs:
  (a) the seven outputs, z_coarse and z_fine are bitwise equal to the evaluation forward's; the saved sigma input is bitwise
      the evaluation kernel's raw sigma + noise * std (FP32, two torch ops); the last sample's saved colour is bitwise the
      background when one is given; every other saved colour is within COLOUR_ULPS FP32 ulps of the float64 sigmoid of
      the evaluation kernel's raw colour.  (The chunked training path renders with the evaluation kernel and
      differentiates a re-run of the training kernel, so the two must agree.)
  (b) every record element of every live sample against tests/torch_reference._mlp in float64 at the kernel's depths
      (sample points formed in FP32 as the kernel forms them, then promoted), decoded at its (unit, pass, tile, row):
        PE image         columns 0-62 within FP16 rounding (2^-11 relative) + PE_ABS[mode]; column 63 is zero
        direction image  columns 0-23 within FP16 rounding + DIR_ABS; columns 24-31 are zero
        activations      exact: |rec - ref| <= 2^-11 |ref| + TAU_EXACT * max|ref of the layer|, per element
                         fast:  max-abs / max|ref| and relative L2 per layer within REC_TOL_FAST
      and the per-sample error of every layer is uniform over the schedule classes of test_render_fp64_gpu.sample_classes
      (CTA iteration 0 / >= 1, pass, tile in the unit, warpgroup half, tile ordinal mod 10: ring slot and parity), KAPPA.
  (c) each ReLU mask bit equals (record element != 0) exactly, everywhere, and equals (float64 pre-activation > 0) wherever
      |a| > MASK_DECIDED[mode] * max|a| of the layer.
  (d) rows that hold no sample (a tile's rows beyond R * S, the rows of an invalid ray in the last unit) are finite in
      every image and zero in the activation images and masks; d raw and every dY image are zero there.

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases and both passes:
  (a) bitwise everywhere; saved colours 2.6 ulps                                   -> COLOUR_ULPS 4
  (b) PE excess over FP16 rounding: exact 2.9e-8, fast 2.8e-7                     -> PE_ABS exact 1e-7, fast 1e-6
      direction image excess: 0                                                   -> DIR_ABS 1e-7
      exact activations, excess over 2^-11 |ref| / max|ref|: 3.0e-6               -> TAU_EXACT 1e-5
      fast activations: max 1.0e-3, L2 7.1e-4                                     -> REC_TOL_FAST (3e-3, 2e-3)
      worst class RMS / overall RMS: exact 1.19, fast 1.11                        -> KAPPA 2.5 (as for the evaluation render)
  (c) undecided mask flips (|a| below the threshold): exact up to 298, fast up to 1.1e5 per case (fast: FP16 weights move
      near-zero pre-activations by up to MASK_DECIDED of the layer's max); none decided
  FP16 range: finite h1 record elements within 2.5e-4 (exact) / 5.9e-4 (fast) of the layer's max; the probe rays'
      layers_xyz.2.weight gradients at 2^14 within 5.9e-4 (exact) / 1.0e-1 (fast) max-abs; non-finite at 1e5 and 4.5e5.
The edges (FP16 range, an empty row beyond the FP16 range, non-finite inputs, state across calls) are described at their
tests.  Defects these tests were checked against, each built once, each caught by the case table (first failing check
given): fast-mode record stores with the two column parities' bases swapped for the second row group of a thread (h0 max
error 0.99 of the layer's max), the mask OR-reduction missing its second shuffle (a0 mask bit against a decided sign), and
the training record pointer one tile back from the CTA's second unit on (direction image off by 1.0).
"""
import types

import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_gpu import REC, decode_image, dev_tensor, dy_off, x_off
from test_backward_fp64_gpu import PROBE_TOL, TOL, errors, grad_pairs, out_grads, reference, rowmap, saved_state, check
from test_render_fp64_gpu import (FAR, NAMES, NEAR, PRECS, dir_cols64, f64, layer1_max, make_case, model, params64,
                                  sample_classes, check_uniformity, schedule, stored_weight, two_iter_rays)

pytestmark = pytest.mark.gpu

H16 = 2.0 ** -11                                   # unit roundoff of FP16
COLOUR_ULPS = 4
PE_ABS = {"exact": 1e-7, "fast": 1e-6}             # sin / cos error of the mode, beyond the FP16 rounding
DIR_ABS = 1e-7
TAU_EXACT = 1e-5
REC_TOL_FAST = (3e-3, 2e-3)                         # (max-abs / max|ref|, relative L2) per layer
MASK_DECIDED = {"exact": 1e-4, "fast": 4e-3}
LAYERS = [(i, f"h{i}", f"a{i}") for i in range(6)] + [(6 + i, f"g{i}", f"a{6 + i}") for i in range(3)]


def width(layer):
    return 256 if layer < 6 else 128


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


def bits(t):
    """The bit pattern of an FP32 tensor (NaN-safe bitwise comparison)."""
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def forward_eval(E, c):
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    out = E.eng.render(c.ro, c.rd, NEAR, FAR, c.nc, c.nf, perturb=c.perturb, noise_std=c.noise_std, white_bkgd=c.white,
                       background=c.bg, dir_z=c.dz, noise=c.noise or None, precision=c.prec, debug=True)
    torch.cuda.synchronize()
    return out


def forward_train(E, c):
    """The training forward; returns its outputs and its saved state (saved_state: depths, records, schedule)."""
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    out = E.eng.render(c.ro, c.rd, NEAR, FAR, c.nc, c.nf, perturb=c.perturb, noise_std=c.noise_std, white_bkgd=c.white,
                       background=c.bg, dir_z=c.dz, noise=c.noise or None, precision=c.prec, train=True)
    s = saved_state(E, c)
    d = s.dbg
    s.raw_c = dev_tensor(d.raw_coarse, (c.n, c.nc, 4)).clone()
    s.raw_f = dev_tensor(d.raw_fine, (c.n, c.nc + c.nf, 4)).clone() if c.nf else None
    s.recs = dev_tensor(d.records, (s.n_tiles, d.record_bytes // 2), "<i2")
    s.maps = [rowmap(c, s, pas) for pas in ((0, 1) if c.nf else (0,))]
    s.used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=E.dev)
    for tile, row in s.maps:
        s.used[tile, row] = True
    return out, s


def masks_of(s):
    m = s.recs.view(torch.uint8)[:, REC["mask"]:REC["mask"] + 9 * 128 * 32].contiguous().view(torch.int32)
    return m.reshape(s.n_tiles, 9, 128, 8)


def mask_bits(masks, layer):
    """[tiles, 128, width] bool: the ReLU mask bits of one layer."""
    m = masks[:, layer]
    b = (m.unsqueeze(-1) >> torch.arange(32, device=m.device, dtype=torch.int32)) & 1
    return b.reshape(m.shape[0], 128, 256)[:, :, :width(layer)].bool()


def taps64(c, p, z, chunk=1 << 16):
    """float64 taps of tests/torch_reference._mlp (pe, ped, a0-a8, h0-h5, g0-g2) at the kernel's depths z [n, S], the sample
    points formed in FP32 like the kernel's (as test_render_fp64_gpu.mlp64); yields (flat sample slice, taps) per chunk."""
    n, S = z.shape
    pts = (c.ro[:, None, :] + c.rd[:, None, :] * z[:, :, None]).reshape(-1, 3)
    dirs = dir_cols64(c)
    expr, lat = f64(c.expr), f64(c.latent)
    for b in range(0, n * S, chunk):
        e = min(n * S, b + chunk)
        ray = torch.arange(b, e, device=z.device) // S
        x = torch.cat((TR._posenc(pts[b:e].double(), 10, True), TR._posenc(dirs[ray], 4, False)), dim=-1).requires_grad_(True)
        taps = {}
        TR._mlp(p, x, expr, lat, taps)  # (x requires grad only so that the taps may retain theirs)
        yield slice(b, e), {k: v.detach() for k, v in taps.items()}


# ---------------------------------------------------------------------------------------------------------------- (a)
def check_against_eval(c, out, s, ev, tag):
    for name in NAMES:
        if name in ev:
            assert same_bits(out[name], ev[name]), (tag, name, "training and evaluation outputs differ")
    assert same_bits(s.z_c, ev["z_coarse"]), (tag, "z_coarse")
    worst_ulps = 0.0
    for key, raw, sfx in (("coarse", s.raw_c, "c"), ("fine", s.raw_f, "f")):
        if raw is None:
            continue
        if key == "fine":
            assert same_bits(s.z_f, ev["z_fine"]), (tag, "z_fine")
        er = ev[f"raw_{key}"]
        sig = er[..., 3] + c.noise[f"n_{sfx}"] * c.noise_std if c.noise_std > 0 else er[..., 3]
        assert same_bits(raw[..., 3], sig), (tag, key, "saved sigma input")
        col = raw[..., :3]
        if c.bg is not None:
            assert same_bits(col[:, -1], c.bg), (tag, key, "saved colour of the last sample")
            col, er = col[:, :-1], er[:, :-1]
        ref = torch.sigmoid(er[..., :3].double())
        ulp = torch.ldexp(torch.ones_like(ref), torch.frexp(ref.float()).exponent - 24)  # FP32 ulp at ref
        ulps = float(((col.double() - ref).abs() / ulp).max())
        worst_ulps = max(worst_ulps, ulps)
        assert ulps <= COLOUR_ULPS, (tag, key, "saved colour", ulps)
    print(f"{tag}: outputs, depths and sigma inputs bitwise equal to the evaluation forward; colours within {worst_ulps:.2f} ulps")


# ---------------------------------------------------------------------------------------------------------------- (b), (c)
def check_records(E, c, s, tag):
    sch = schedule(E, c)
    masks = masks_of(s)
    W = {"max_ref": [0.0] * 9, "excess": [0.0] * 9, "dmax": [0.0] * 9, "d2": [0.0] * 9, "r2": [0.0] * 9}
    sq = [[] for _ in range(9)]
    cls = []
    flips = undecided = 0
    pe_worst = dir_worst = 0.0
    amax = [0.0] * 9
    passes = [(0, "coarse", c.mc, s.z_c)] + ([(1, "fine", c.mf, s.z_f)] if c.nf else [])
    for pas, key, m, z in passes:
        tile, row = s.maps[pas]
        p = params64(m)
        pe = decode_image(s.recs, REC["pe"][0], 64)
        ped = decode_image(s.recs, REC["ped"][0], 32)
        assert float(pe[:, :, 63].abs().max()) == 0.0 and float(ped[:, :, 24:].abs().max()) == 0.0, (tag, "padding columns")
        pe, ped = pe[tile, row], ped[tile, row]
        imgs = [decode_image(s.recs, x_off(L), width(L))[tile, row] for L in range(9)]
        bitsl = [mask_bits(masks, L)[tile, row] for L in range(9)]
        for sl, t in taps64(c, p, z):
            e = (pe[sl, :63].double() - t["pe"]).abs() - H16 * t["pe"].abs()
            pe_worst = max(pe_worst, float(e.max()))
            e = (ped[sl, :24].double() - t["ped"]).abs() - H16 * t["ped"].abs()
            dir_worst = max(dir_worst, float(e.max()))
            for L, hname, aname in LAYERS:
                got, ref = imgs[L][sl].double(), t[hname]
                assert bool(torch.isfinite(got).all()), (tag, key, hname, "non-finite record")
                d = got - ref
                W["max_ref"][L] = max(W["max_ref"][L], float(ref.abs().max()))
                W["excess"][L] = max(W["excess"][L], float((d.abs() - H16 * ref.abs()).max()))
                W["dmax"][L] = max(W["dmax"][L], float(d.abs().max()))
                W["d2"][L] += float(d.pow(2).sum())
                W["r2"][L] += float(ref.pow(2).sum())
                sq[L].append(d.pow(2).sum(-1))
                a = t[aname]
                amax[L] = max(amax[L], float(a.abs().max()))
                # sign of the pre-activation: judged once the layer's max is known (kept per chunk as (|a|, flip))
                flip = bitsl[L][sl] != (a > 0)
                if bool(flip.any()):
                    W.setdefault("flips", []).append((L, a.abs()[flip]))
        cls.append(sample_classes(E, c, sch, pas))
    assert pe_worst <= PE_ABS[c.prec] and dir_worst <= DIR_ABS, (tag, pe_worst, dir_worst)
    cls = torch.cat(cls)
    worst_rec, worst_cls = [0.0, 0.0], 0.0
    for L, hname, _ in LAYERS:
        mx = W["max_ref"][L]
        if c.prec == "exact":
            rel = W["excess"][L] / mx
            worst_rec[0] = max(worst_rec[0], rel)
            assert rel <= TAU_EXACT, (tag, hname, rel)
        else:
            em, el = W["dmax"][L] / mx, (W["d2"][L] / W["r2"][L]) ** 0.5
            worst_rec = [max(worst_rec[0], em), max(worst_rec[1], el)]
            assert em <= REC_TOL_FAST[0] and el <= REC_TOL_FAST[1], (tag, hname, em, el)
        worst_cls = max(worst_cls, check_uniformity(f"{tag} {hname}", torch.cat(sq[L]), cls))
    for L, mag in W.get("flips", []):
        decided = mag > MASK_DECIDED[c.prec] * amax[L]
        assert not bool(decided.any()), (tag, f"a{L}", "mask bit against a decided sign", float(mag.max()) / amax[L])
        undecided += int(mag.numel())
    # every mask bit is (record element != 0), at every row of every tile
    for L in range(9):
        img = decode_image(s.recs, x_off(L), width(L))
        assert torch.equal(mask_bits(masks, L), bits(img) != 0), (tag, L, "mask bit differs from its record element")
    print(f"{tag} records: PE excess {pe_worst:.1e}, direction excess {dir_worst:.1e}, activations "
          + (f"worst excess / max {worst_rec[0]:.2e}" if c.prec == "exact" else f"worst max {worst_rec[0]:.2e}, L2 {worst_rec[1]:.2e}")
          + f"; worst class RMS / overall {worst_cls:.2f}; {undecided} undecided mask flips")


# ---------------------------------------------------------------------------------------------------------------- (d)
def check_empty_rows(E, c, s, tag):
    """Finite everywhere, activation images and masks zero in rows that hold no sample; d raw and dY zero there after a
    backward."""
    dead = ~s.used
    n_dead = int(dead.sum())
    for off, w in [(REC["pe"][0], 64), (REC["ped"][0], 32)] + [(x_off(L), width(L)) for L in range(9)]:
        img = decode_image(s.recs, off, w)
        assert bool(torch.isfinite(img[dead]).all()), (tag, off, "non-finite record in a row without a sample")
    masks = masks_of(s)
    for L in range(9):
        assert float(decode_image(s.recs, x_off(L), width(L))[dead].abs().max() if n_dead else 0.0) == 0.0, (tag, L)
        assert not bool(mask_bits(masks, L)[dead].any()), (tag, L, "mask bit in a row without a sample")
    kernel_backward(E, c, out_grads(E, c, seed=31))
    d_raw = dev_tensor(s.dbg.d_raw, (s.n_tiles, 128, 4))
    assert float(d_raw[dead].abs().max() if n_dead else 0.0) == 0.0, (tag, "d raw")
    for L in range(9):
        dy = decode_image(s.recs, dy_off(L), width(L))
        assert float(dy[dead].abs().max() if n_dead else 0.0) == 0.0, (tag, L, "dY in a row without a sample")
    print(f"{tag}: {n_dead} rows without a sample, zero in every activation image, mask, d raw and dY")


def kernel_backward(E, c, gouts, inputs=None):
    pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
    pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER] if c.mf is not None else None
    r = E.eng.backward(list(gouts), pc, pf, inputs=inputs)
    torch.cuda.synchronize()
    return r


# ---------------------------------------------------------------------------------------------------------------- cases
def _prod(stress):
    return lambda E, prec: make_case(E, 2048, 64, 64, prec, stress=stress, perturb=True, noise_std=0.1, seed=50)


def _counts(nc, nf):
    return lambda E, prec: make_case(E, two_iter_rays(E), nc, nf, prec, perturb=True, noise_std=0.1, seed=nc + nf)


def _opt(**kw):
    return lambda E, prec: make_case(E, two_iter_rays(E), 64, 64, prec, seed=7, **kw)


CASES = {
    # 2048 rays at 64c+64f: 1024 units, 3072 tiles, every CTA runs 7-8 units
    "prod2048_random_init": _prod(False),
    "prod2048_stress": _prod(True),
    # 4 * SMs + 37 rays: every CTA runs at least two units, the last unit is half filled (an invalid ray)
    "64c128f": _counts(64, 128),
    "100c60f": _counts(100, 60),       # rays straddle tiles; partly filled last tiles
    "256c256f": _counts(256, 256),     # one ray per unit
    "64c0f": _counts(64, 0),
    "3c0f": _counts(3, 0),             # 6 of 128 rows hold a sample
    # options
    "white_nobg": _opt(white=True, bg=False),
    "nobg": _opt(bg=False),
    "dir_z": _opt(dir_z=True),
    # 1, 2 and 3 rays: idle CTAs, a partly valid unit
    "1ray": lambda E, prec: make_case(E, 1, 64, 128, prec, seed=1),
    "2rays": lambda E, prec: make_case(E, 2, 64, 128, prec, seed=2),
    "3rays": lambda E, prec: make_case(E, 3, 64, 128, prec, seed=3),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(CASES))
def test_training_forward_against_float64(E, case, prec):
    c = CASES[case](E, prec)
    tag = f"{case} {prec}"
    ev = forward_eval(E, c)
    out, s = forward_train(E, c)
    check_against_eval(c, out, s, ev, tag)
    check_records(E, c, s, tag)
    check_empty_rows(E, c, s, tag)


# ---------------------------------------------------------------------------------------------------------------- FP16 range
@pytest.mark.parametrize("prec", PRECS)
def test_fp16_range_of_saved_activations(E, prec):
    """The gain construction of test_fp16_range_of_hidden_activations (layers_xyz.1 x g, layers_xyz.2's weight / g; the
    reference uses layers_xyz.2's weight as the kernel stores it) with the largest h1 at 2^14, 1e5 and 4.5e5.  Every element
    of the h1 record of every live sample is within tolerance of float64 or non-finite, never finite and wrong.  The ray
    holding the largest h1 of each network then gets an output gradient alone: that network's layers_xyz.2.weight gradient
    (formed from the h1 record) is non-finite or within PROBE_TOL of float64.  The other gradients go through W2^T, deep in
    FP16's subnormal range at these gains, and are not judged."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=30)
    base = forward_eval(E, c)
    nets = {"coarse": c.mc, "fine": c.mf}
    amax = {key: float(layer1_max(c, params64(m), base[f"z_{key}"])[0].max()) for key, m in nets.items()}
    for target in (2.0 ** 14, 1.0e5, 4.5e5):
        models, refp, refm = {}, {}, {}
        for key, m in nets.items():
            g = target / amax[key]
            p = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
            p["layers_xyz.1.weight"] *= g
            p["layers_xyz.1.bias"] *= g
            p["layers_xyz.2.weight"] /= g
            models[key] = model(E, 0, True, params=p)
            w2 = dict(models[key].named_parameters())["layers_xyz.2.weight"].detach()
            refp[key] = params64(models[key], {"layers_xyz.2.weight": stored_weight(w2, prec)})
            q = dict(p)
            q["layers_xyz.2.weight"] = stored_weight(w2, prec).float().cpu()
            refm[key] = model(E, 0, True, params=q)
        c2 = types.SimpleNamespace(**vars(c))
        c2.mc, c2.mf = models["coarse"], models["fine"]
        out, s = forward_train(E, c2)
        n_nonfinite, worst = 0, 0.0
        probe = {}
        for pas, key in ((0, "coarse"), (1, "fine")):
            z = s.z_f if pas else s.z_c
            tile, row = s.maps[pas]
            got = decode_image(s.recs, x_off(1), 256)[tile, row].double()
            ref = torch.cat([t["h1"] for _, t in taps64(c2, refp[key], z)])
            mx = float(ref[torch.isfinite(ref)].abs().max())
            err = (got - ref).abs()
            bound = H16 * ref.abs() + (TAU_EXACT if prec == "exact" else REC_TOL_FAST[0]) * mx
            fin = torch.isfinite(got)
            bad = fin & ~(err <= bound)
            assert not bool(bad.any()), (prec, target, key, "finite and wrong h1 record", int(bad.sum()),
                                         float(got[bad].abs().max()), float(ref[bad].abs().max()))
            n_nonfinite += int((~fin).sum())
            worst = max(worst, float((err[fin] / mx).max()))
            probe[key] = int(ref.abs().amax(-1).nan_to_num(0.0).argmax()) // z.shape[1]
        # output gradients on the probe ray of each network only (the coarse network sees only coarse outputs)
        dense = out_grads(E, c2, seed=32)
        gouts = []
        for i, t in enumerate(dense):
            zt = torch.zeros_like(t)
            ray = probe["coarse"] if i < 3 else probe["fine"]
            zt[ray] = t[ray] * c.n
            gouts.append(zt)
        kg = kernel_backward(E, c2, gouts)
        cr = types.SimpleNamespace(**vars(c2))
        cr.mc, cr.mf = refm["coarse"], refm["fine"]
        verdict = []
        for key, idx in (("coarse", 0), ("fine", 1)):
            R = reference(E, cr, s.z_c, s.z_f, gouts, lo=probe[key], hi=probe[key] + 1)
            g = kg[idx][TR.PARAM_ORDER.index("layers_xyz.2.weight")]
            r = (R.gc if idx == 0 else R.gf)[TR.PARAM_ORDER.index("layers_xyz.2.weight")]
            if not bool(torch.isfinite(g).all()):
                verdict.append(f"{key} non-finite")
                continue
            em, el = errors(g, r)
            verdict.append(f"{key} max {em:.2e} L2 {el:.2e}")
            assert em <= PROBE_TOL[prec][0] and el <= PROBE_TOL[prec][1], (prec, target, key, "finite, wrong dW2", em, el)
        print(f"{prec} max h1 -> {target:.3g}: {n_nonfinite} non-finite h1 record elements, worst finite error {worst:.2e}; "
              f"layers_xyz.2.weight gradient of the probe rays: {', '.join(verdict)}")


# ---------------------------------------------------------------------------------------------------------------- empty rows
@pytest.mark.parametrize("prec", PRECS)
def test_empty_row_beyond_fp16_range(E, prec):
    """Weights whose layer-0 unit j is zero (pre-activation <= -2) at every live sample but +2 at the camera origin, where
    the rows beyond R * S of a tile evaluate (ray 0 of the unit at z = 0), and layers_xyz.1 weight 5e4 on that unit: h1 of
    those rows is about 1e5, beyond FP16.  100c+60f leaves 56 and 64 such rows per unit; the odd ray count leaves an invalid
    ray.  The float64 gradients are finite (no reference evaluates those rows), so the kernel's must be finite and within
    the dense tolerance of test_backward_fp64_gpu."""
    c = make_case(E, two_iter_rays(E), 100, 60, prec, perturb=True, noise_std=0.1, seed=33)
    assert c.n % 2 == 1
    # s(p) = u . p with u against the mean ray direction: largest at the origins, smaller at every sample (z >= near)
    u = -c.rd.double().mean(0)
    u = u / u.norm()
    s_origin = float((c.ro.double() @ u).min())
    s_live = float((c.ro.double() @ u + NEAR * (c.rd.double() @ u)).max())
    gap = s_origin - s_live
    assert gap > 0.0, gap
    thr = s_live + 0.5 * gap
    A = 2.0 / (0.5 * gap)                      # pre-activation A (s - thr): >= +2 at an origin, <= -2 at every sample
    j, k = 17, 40

    def edit(m):
        p = {key: v.detach().cpu().clone() for key, v in m.state_dict().items()}
        p["layers_xyz.0.weight"][j] = 0.0
        p["layers_xyz.0.weight"][j, :3] = (A * u).float().cpu()
        p["layers_xyz.0.bias"][j] = -A * thr
        p["layers_xyz.1.weight"][k, j] = 5.0e4
        return model(E, 0, True, params=p)
    c.mc, c.mf = edit(c.mc), edit(c.mf)
    out, s = forward_train(E, c)
    # the construction: unit j is off at every live sample (float64), on at the origin
    for pas, key, m, z in ((0, "coarse", c.mc, s.z_c), (1, "fine", c.mf, s.z_f)):
        a0 = torch.cat([t["a0"][:, j] for _, t in taps64(c, params64(m), z)])
        assert float(a0.max()) <= -1.0, (key, float(a0.max()))
    gouts = out_grads(E, c, seed=34)
    kg = kernel_backward(E, c, gouts)
    R = reference(E, c, s.z_c, s.z_f, gouts)
    nonfin = [name for name, g, _ in grad_pairs(kg, R) if not bool(torch.isfinite(g).all())]
    print(f"{prec}: {int((~s.used).sum())} rows without a sample; non-finite kernel gradients: {nonfin or 'none'}")
    check(f"empty rows beyond FP16 {prec}", grad_pairs(kg, R), TOL[prec])


# ---------------------------------------------------------------------------------------------------------------- non-finite
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("field", ["origin", "background", "sigma_noise", "weight", "expression"])
def test_nonfinite_inputs_in_training(E, field, bad, prec):
    """A NaN or +inf in one ray's origin, background or sigma-noise draw, in one layers_xyz.1 weight or in the expression.
    The training forward's outputs equal the evaluation forward's bit for bit, non-finite entries included.  After
    nfb_loss_mse_grad and the backward, every gradient float64 autograd makes non-finite is non-finite; for the per-ray
    inputs every other ray's origin, direction and background gradients are finite and match the clean run's (the loss
    scale skips non-finite rays).  A NaN ReLU input of sigma passes its gradient, as in torch (fc_alpha.bias is NaN)."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, perturb=True, noise_std=0.1, seed=40)
    ray = c.n // 2 + 1
    v = float(bad)
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
    else:
        d.expr = c.expr.clone()
        d.expr[3] = v
    per_ray = field in ("origin", "background", "sigma_noise")
    inputs = ("ray_origins", "ray_directions", "background")
    target = torch.rand(c.n, 3, generator=torch.Generator().manual_seed(41)).to(E.dev)

    def run(cc):
        ev = forward_eval(E, cc)
        out, s = forward_train(E, cc)
        for name in NAMES:
            assert same_bits(out[name], ev[name]), (field, bad, name, "training and evaluation outputs differ")
        gc, gf = torch.zeros(c.n, 3, device=E.dev), torch.zeros(c.n, 3, device=E.dev)
        E.eng.loss_mse_grad(out["rgb_coarse"], out["rgb_fine"], target, c.n, gc, gf, torch.zeros(2, device=E.dev))
        gouts = [gc, None, None, gf, None, None, None]
        return out, s, gouts, kernel_backward(E, cc, gouts, inputs=inputs if per_ray else None)

    _, _, _, clean = run(c)
    out, s, gouts, kg = run(d)
    lo, hi = (ray, ray + 1) if per_ray else (0, 8)
    R = reference(E, d, s.z_c, s.z_f, gouts, lo=lo, hi=hi)
    reached = 0
    for name, g, r in grad_pairs(kg[:3], R):
        nonfin = ~torch.isfinite(r)
        reached += int(nonfin.sum())
        assert bool((~torch.isfinite(g[nonfin])).all()), (field, bad, name, "finite where torch gives a non-finite gradient")
    if per_ray:
        others = torch.ones(c.n, dtype=torch.bool, device=E.dev)
        others[ray] = False
        for name in inputs:
            g, g0 = kg[3][name][others], clean[3][name][others]
            assert bool(torch.isfinite(g).all()), (field, bad, name, "another ray's input gradient is non-finite")
            # the bad ray can change the power-of-two loss scale, which moves only FP16 subnormals of the chain (measured
            # 2.4e-6 with an inf sigma-noise draw, otherwise 0)
            err = float((g - g0).abs().max()) / float(g0.abs().max())
            assert err <= 2e-5, (field, bad, name, err)
    print(f"{field} = {bad} ({prec}): {reached} gradient entries non-finite in float64 autograd, all non-finite in the kernel")


# ---------------------------------------------------------------------------------------------------------------- state
@pytest.mark.parametrize("prec", PRECS)
def test_no_state_leaks_across_calls(E, prec, monkeypatch):
    """With a fixed memory budget (so the chunk plan does not follow free memory): a clean training call and its backward,
    a call with a NaN origin at a larger batch and its backward, then the first call again: its outputs, the records of
    its live rows and its gradients equal the first call's bit for bit."""
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "4096")
    a = make_case(E, two_iter_rays(E), 64, 64, prec, perturb=True, noise_std=0.1, seed=42)
    b = make_case(E, 2048, 64, 64, prec, perturb=True, noise_std=0.1, seed=43)
    b.ro = b.ro.clone()
    b.ro[5, 2] = float("nan")
    images = [(REC["pe"][0], 64), (REC["ped"][0], 32)] + [(x_off(L), width(L)) for L in range(9)] \
        + [(dy_off(L), width(L)) for L in range(9)]

    def run(cc):
        out, s = forward_train(E, cc)
        kg = kernel_backward(E, cc, out_grads(E, cc, seed=44))
        recs = [torch.cat([decode_image(s.recs, off, w)[tile, row] for tile, row in s.maps]) for off, w in images]
        return [out[k].clone() for k in NAMES], recs, [t for t in list(kg[0]) + list(kg[1]) + [kg[2]] if t is not None]

    first = run(a)
    run(b)
    again = run(a)
    for what, x, y in zip(("outputs", "records", "gradients"), first, again):
        for i, (p, q) in enumerate(zip(x, y)):
            assert same_bits(p, q), (prec, what, i)
    print(f"{prec}: a clean call after a NaN call at 2048 rays repeats the first call bit for bit")
