"""Exact-grad mode (NFB_PREC_EXACT_GRAD, include/nfb.h): exact mode's forward and a backward on hi + lo operands end to end.

(a) pack      the lo half of the backward stream (NfbWeightDebug.bwd_lo) is, byte for byte, the transposition of the lo units of
              the x3 stream (tests/weight_pack_reference.py's Layout names the weight every slot holds); x1, x3 and bwd are the
              bytes of a handle that never ran exact-grad; nfb_load_weights keeps the lo half current.
(b) forward   outputs and the forward's part of every record (PE, h0..h5, g0..g2, PEd, masks) equal exact mode's bit for bit,
              single- and multi-frame, at several sample counts with perturbation, noise, background and dir_z; the lo images
              bring hi + lo to the float64 activation: error(hi + lo) <= LO_GAIN * error(hi alone); PE and PEd against float64
              encodings of the kernel's own FP32 points and direction inputs, PE_LO_GAIN.
(c) float64   end to end: all 48 parameter gradients and the latent against tests/torch_reference.py in float64
              (tests/test_backward_fp64_gpu.py's reference and error measures): dense 2048 rays, the stress weights, 3c+0f, dir_z
              on a white background, single rays, the chunked path and the input-only latent; per-ray input gradients and d
              expression; F = 5 frames (per-frame latents and expressions, inputs, parameters).  Every case also runs exact mode.
              Then every path of the backward at the kernel's OWN forward state (its d raw, masks and hi + lo activations), RATIO
              times below exact mode: all accumulator blocks of the full launch, the PE-only launch, the input-gradient rows and the
              per-ray and per-frame sums of a multi-frame backward.
(d) rules     two backwards repeat bit for bit, and a NaN input / an activation beyond the FP16 range gives non-finite gradients.

Measured on an H100 80GB HBM3 (CUDA 12.9), worst tensor per case, (max, L2) relative error, exact -> exact-grad:
  dense 2048r 64c+64f     7.5e-4, 5.3e-4 -> 1.9e-4, 1.6e-4   (4x, 3x)
  stress 64c+128f         6.1e-4, 5.4e-4 -> 1.6e-4, 1.2e-4   (4x, 5x)
  3c+0f                   7.9e-4, 7.4e-4 -> 5.5e-5, 5.5e-5   (14x, 13x)
  dir_z white 100c+60f    6.0e-4, 5.6e-4 -> 3.6e-4, 1.9e-4   (2x, 3x)
  single rays             8.5e-4, 7.2e-4 -> 1.3e-5, 1.2e-5   (68x, 59x)
  chunked                 5.7e-4, 6.2e-4 -> 2.5e-4, 2.7e-4   (2x, 2x)
  input-only latent       4.2e-4, 4.7e-4 -> 2.9e-4, 2.6e-4   (1.5x, 2x)                -> E2E_TOL (1e-3, 5e-4), E2E_RATIO 1
  inputs + expression     5.8e-3, 1.7e-3 -> 5.6e-3, 1.6e-3   (1x)                      -> IN_E2E_TOL (2e-2, 6e-3)
  F = 5 frames            2.1e-2, 4.2e-3 -> 2.1e-2, 4.2e-3   (1x)                      -> MF_E2E_TOL (5e-2, 1e-2)
  at the kernel's state (64c+64f / 64c+0f / 64c+64f F = 5), exact -> exact-grad worst max:
    accumulators, full launch   6.1e-4 -> 5.2e-5 (12x, L2 15x) / 5.5e-4 -> 1.6e-5 (34x) / 6.6e-4 -> 5.2e-5 (13x, L2 15x)
    PE-only launch              5.2e-4 -> 1.1e-5 (48x) / 5.3e-4 -> 7.0e-6 (76x)
    input-gradient rows         7.0e-4 -> 4.5e-6 (156x) / 5.0e-4 -> 3.6e-6 (139x) / 6.9e-4 -> 3.1e-6 (219x)
    per-ray / per-frame sums    3.9e-4 -> 2.9e-6 (134x) / 3.5e-4 -> 2.8e-6 (128x)       -> STATE_TOL (1e-4, 1e-4), RATIO 10
  lo images               error(hi + lo) / error(hi) against float64 at most 2.3e-2       -> LO_GAIN 0.1
  PE, PEd lo              at most 6.0e-4                                                  -> PE_LO_GAIN 1e-2
End to end, exact-grad's error is bounded by the forward it shares with exact mode: d raw comes from the forward's FP32 state
(colours, sigma inputs, ReLU branches within the forward's rounding of zero), which differs from float64 by ~1e-5 and moves
dense gradients by ~1e-4 (test_backward_fp64_gpu.py measures d raw's L2 error at 8.3e-4 in exact mode).  Where that state
agrees with float64 (single rays, the kernel's own state) the backward's own error is 3e-6 to 5e-5, 12-220x below exact
mode's.  Per-ray input gradients end to end are dominated the same way (sin / cos of the 2^9 frequency at the forward's FP32
point), so there exact-grad matches exact mode, and the stages at the kernel's state carry the comparison.
"""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
import weight_pack_reference as WP
from test_backward_fp64_gpu import (NAMES, errors, grad_pairs, kernel_backward, make_case, out_grads, reference, rowmap,
                                    saved_state, train_forward, two_iter_rays)
from test_backward_gpu import decode_image, dev_tensor, x_off

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E(built_lib):
    """test_backward_fp64_gpu.py's case environment with a renderer handle of this module's own: an exact-grad training forward
    switches a handle to re-packing the lo stream too (one more launch per re-pack), which the shared handle must not see."""
    import nerf
    from nerf import _capi, _engine
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    e = types.SimpleNamespace(nerf=nerf, capi=_capi, dev=torch.device("cuda", 0))
    e.eng = _engine.Renderer(e.dev)
    e.sms = torch.cuda.get_device_properties(0).multi_processor_count
    fr = O.synthetic_frame(21, 48, 48)
    ro, rd = O.ray_bundle(48, 48, fr["intrinsics"], fr["pose"])
    e.ro, e.rd = ro.reshape(-1, 3).to(e.dev), rd.reshape(-1, 3).to(e.dev)
    e.bg = fr["bg"].reshape(-1, 3).to(e.dev)
    e.expr, e.latent = fr["expr"].to(e.dev), fr["latent"].to(e.dev)
    e._models = {}
    return e

MIB = 1 << 20
PED_OFF = 16384 + 6 * 65536 + 3 * 32768                         # nfb_layout.h kRecPEd
REC_DY0 = PED_OFF + 8192 + 9 * 128 * 32                          # nfb_layout.h kRecDY0: the forward writes the bytes below it
E2E_TOL = (1e-3, 5e-4)   # (max, L2) of the exact-grad parameter gradients against float64, relative to the tensor's max / norm
E2E_RATIO = 1.0          # exact's worst error over exact-grad's, at least, end to end (bounded by the forward's error, see above)
IN_E2E_TOL = (2e-2, 6e-3)  # per-ray input and expression gradients end to end (exact mode's IN_TOL)
MF_E2E_TOL = (5e-2, 1e-2)  # F = 5: per-frame latent / expression, per-ray input and parameter gradients end to end
STATE_TOL = (1e-4, 1e-4) # (max, L2) against float64 at the kernel's own forward state, every category
RATIO = 10.0             # exact's worst error over exact-grad's there, at least
LO_GAIN = 0.1            # error of hi + lo over the error of hi alone, activations against float64
PE_LO_GAIN = 0.01        # the same for PE and PEd against float64 encodings of the kernel's FP32 points


def weights(E, net):
    return E.eng.weights_debug(net)


def dev_bytes(ptr, n):
    return dev_tensor(ptr, (n,), "|u1").clone().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------- (a)
def test_bwd_lo_is_the_transposed_lo_of_x3(E):
    from nerf import _engine
    c = make_case(E, 64, 64, 64, "exact_grad", seed=1)
    layout = WP.Layout(E.capi.lib)
    src_lo = layout.x3[layout.x3_lo_slot]
    order = np.argsort(src_lo, kind="stable")
    fresh = _engine.Renderer(E.dev)  # never runs exact-grad
    fresh.sync_weights(c.mc, c.mf)
    for step, m in enumerate((c.mc, model_other(E))):
        if step:
            E.eng.sync_weights(m, c.mf)  # nfb_load_weights of the coarse network after the flag: the lo half follows
            fresh.sync_weights(m, c.mf)
        else:
            train_forward(E, c)  # the first exact-grad training forward builds the lo half of the loaded streams
        torch.cuda.synchronize()
        for net in (0, 1):
            w, f = weights(E, net), fresh.weights_debug(net)
            assert w.bwd_lo and w.bwd_lo_bytes == w.bwd_bytes and not f.bwd_lo and f.bwd_lo_bytes == 0
            for name in ("x1", "x3", "bwd"):
                n = getattr(w, name + "_bytes")
                assert np.array_equal(dev_bytes(getattr(w, name), n), dev_bytes(getattr(f, name), n)), (net, name)
            x3 = dev_bytes(w.x3, w.x3_bytes).view(np.uint16)
            lo = dev_bytes(w.bwd_lo, w.bwd_lo_bytes).view(np.uint16)
            want = np.zeros_like(lo)
            has = layout.bwd >= 0
            pos = np.searchsorted(src_lo[order], layout.bwd[has])
            assert np.array_equal(src_lo[order][pos], layout.bwd[has])  # every weight of bwd has a lo unit entry in x3
            want[has] = x3[layout.x3_lo_slot[order][pos]]
            assert (layout.bwd >= -1).all()  # every slot of bwd belongs to a unit
            assert np.array_equal(lo, want), (step, net, int((lo != want).sum()))
            assert int(np.count_nonzero(lo)) > lo.size // 4  # the lo half is populated


def model_other(E):
    from test_backward_fp64_gpu import model
    return model(E, 333, True)


# ---------------------------------------------------------------------------------------------------------------- (b)
FWD_CASES = {"64c128f": dict(nc=64, nf=128), "128c256f": dict(nc=128, nf=256), "3c7f": dict(nc=3, nf=7),
             "64c0f": dict(nc=64, nf=0), "64c128f_dirz_white": dict(nc=64, nf=128, dir_z=True, white=True, bg=False)}


def records(E, n_tiles, stride):
    d = E.eng.train_debug()
    assert d.record_bytes == stride and d.n_tiles == n_tiles
    return dev_tensor(d.records, (n_tiles, stride), "|u1").clone()


@pytest.mark.parametrize("case", list(FWD_CASES))
def test_forward_is_exact_modes(E, case):
    kw = dict(FWD_CASES[case])
    nc, nf = kw.pop("nc"), kw.pop("nf")
    c = make_case(E, two_iter_rays(E), nc, nf, "exact", seed=nc + nf, **kw)
    out_x = train_forward(E, c)
    s = saved_state(E, c)
    rec_x = records(E, s.n_tiles, MIB)
    c.prec = "exact_grad"
    out_g = train_forward(E, c)
    rec_g = records(E, s.n_tiles, 2 * MIB)
    for k in NAMES:
        if out_x.get(k) is not None:
            assert torch.equal(out_x[k], out_g[k]), (case, k)
    assert torch.equal(rec_x[:, :REC_DY0], rec_g[:, :REC_DY0]), case
    # the lo images: hi + lo against the float64 activations of the reference at the kernel's depths
    n = min(c.n, 64)
    f64 = lambda t: None if t is None else t.detach().to(E.dev, torch.float64)  # noqa: E731
    pc = {k: f64(v).requires_grad_(True) for k, v in c.mc.named_parameters()}  # the taps retain gradients
    pf = {k: f64(v).requires_grad_(True) for k, v in c.mf.named_parameters()} if c.mf is not None else None
    rays = torch.cat((c.ro[:n], c.rd[:n], torch.full((n, 1), 0.2, device=E.dev), torch.full((n, 1), 0.8, device=E.dev)), -1).double()
    taps = {}
    TR.render_at_depths(rays, pc, pf, f64(c.expr), f64(c.latent), f64(s.z_c[:n]), f64(s.z_f[:n]) if s.z_f is not None else None,
                        0.2, 0.8, c.noise_std, {k: f64(v[:n]) for k, v in c.noise.items()}, c.white,
                        f64(c.bg[:n]) if c.bg is not None else None, f64(c.dz[:n]) if c.dz is not None else None, taps)
    i16 = rec_g.view(torch.int16)
    hi16, lo16 = i16[:, :MIB // 2].contiguous(), i16[:, MIB // 2:].contiguous()
    worst = 0.0
    for pas, key in ((0, "coarse"), (1, "fine")):
        if key not in taps:
            continue
        tile, row = rowmap(c, s, pas)
        Sx = c.nc + c.nf if pas else c.nc
        tile, row = tile[:n * Sx], row[:n * Sx]
        for L in range(9):
            W = 256 if L < 6 else 128
            ref = taps[key][f"h{L}" if L < 6 else f"g{L - 6}"].reshape(-1, W)
            hi = decode_image(hi16, x_off(L), W)[tile, row].double()
            lo = decode_image(lo16, x_off(L), W)[tile, row].double()
            ref = ref.detach()
            e_hi, e_hl = float((hi - ref).abs().max()), float((hi + lo - ref).abs().max())
            if e_hi > 0:
                worst = max(worst, e_hl / e_hi)
            assert e_hl <= LO_GAIN * e_hi + 1e-6 * float(ref.abs().max()), (case, key, L, e_hi, e_hl)
    # PE and PEd against float64 of the encodings at the kernel's own FP32 inputs: the point fl(o + fl(d z)) and the direction
    # input (dir_z or d_z, near, far), each frequency an exact power-of-two multiple, sin / cos in float64
    pe_worst = 0.0
    for pas in range(2 if c.nf else 1):
        tile, row = rowmap(c, s, pas)
        Sx = c.nc + c.nf if pas else c.nc
        z = (s.z_f if pas else s.z_c)
        pt = (c.ro[:, None, :] + c.rd[:, None, :] * z[..., None]).reshape(-1, 3).double()
        f = 2.0 ** torch.arange(10, dtype=torch.float64, device=E.dev)
        xs = pt[:, None, :] * f[None, :, None]
        pe = torch.cat((pt, torch.cat((torch.sin(xs), torch.cos(xs)), 2).reshape(-1, 60), torch.zeros_like(pt[:, :1])), 1)
        v0 = (c.dz if c.dz is not None else c.rd[:, 2]).float()
        v = torch.stack((v0, torch.full_like(v0, 0.2), torch.full_like(v0, 0.8)), 1).double()
        xd = v[:, None, :] * (2.0 ** torch.arange(4, dtype=torch.float64, device=E.dev))[None, :, None]
        ped = torch.cat((torch.cat((torch.sin(xd), torch.cos(xd)), 2).reshape(-1, 24), torch.zeros(c.n, 8, dtype=torch.float64,
                                                                                                     device=E.dev)), 1)
        ped = ped[:, None, :].expand(c.n, Sx, 32).reshape(-1, 32)
        for name, off, W, ref in (("PE", 0, 64, pe), ("PEd", PED_OFF, 32, ped)):
            hi = decode_image(hi16, off, W)[tile, row].double()
            lo = decode_image(lo16, off, W)[tile, row].double()
            e_hi, e_hl = float((hi - ref).abs().max()), float((hi + lo - ref).abs().max())
            pe_worst = max(pe_worst, e_hl / e_hi)
            assert e_hl <= PE_LO_GAIN * e_hi, (case, name, pas, e_hi, e_hl)
    print(f"{case}: worst error(hi + lo) / error(hi) over the activation images {worst:.2e}, over PE and PEd {pe_worst:.2e}")


def test_multi_frame_forward_is_exact_modes(E):
    c = make_case(E, two_iter_rays(E), 64, 128, "exact", seed=5, dir_z=True)
    F = 5
    g = torch.Generator().manual_seed(3)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames((torch.rand(F, 76, generator=g) - 0.5).to(E.dev), (torch.rand(F, 32, generator=g) - 0.5).to(E.dev))
    fi = (torch.arange(c.n) % F).to(E.dev)
    outs, recs = [], []
    for prec, stride in (("exact", MIB), ("exact_grad", 2 * MIB)):
        o = E.eng.render(c.ro, c.rd, 0.2, 0.8, c.nc, c.nf, perturb=True, noise_std=0.1, background=c.bg, dir_z=c.dz, noise=c.noise,
                         precision=prec, train=True, frame_index=fi)
        torch.cuda.synchronize()
        d = E.eng.train_debug()
        outs.append({k: o[k].clone() for k in NAMES if torch.is_tensor(o.get(k))})
        recs.append(records(E, int(d.n_tiles), stride)[:, :REC_DY0])
    assert outs[0].keys() == outs[1].keys() and len(outs[0]) == len(NAMES)
    for k in NAMES:
        assert torch.equal(outs[0][k], outs[1][k]), k
    assert torch.equal(recs[0], recs[1])


# ---------------------------------------------------------------------------------------------------------------- (c)
def worst(pairs):
    em = max(errors(g, r)[0] for _, g, r in pairs)
    el = max(errors(g, r)[1] for _, g, r in pairs)
    return em, el


def compare(tag, runs, tol=E2E_TOL):
    """runs: prec -> list of (name, kernel gradient, float64 gradient).  Exact-grad within tol, and no worse than exact."""
    (xm, xl), (gm, gl) = worst(runs["exact"]), worst(runs["exact_grad"])
    print(f"{tag}: exact max {xm:.2e} L2 {xl:.2e}; exact_grad max {gm:.2e} L2 {gl:.2e}; ratio {xm / max(gm, 1e-30):.0f}x, "
          f"{xl / max(gl, 1e-30):.0f}x")
    for _, g, _ in runs["exact_grad"]:
        assert bool(torch.isfinite(g).all()), tag
    assert gm <= tol[0] and gl <= tol[1], (tag, gm, gl)
    assert gm * E2E_RATIO <= xm and gl * E2E_RATIO <= xl, (tag, xm, gm, xl, gl)


E2E_CASES = {"dense_2048r_64c64f": dict(n=2048, nc=64, nf=64, stress=False),
             "stress_64c128f": dict(n=None, nc=64, nf=128),
             "3c0f": dict(n=None, nc=3, nf=0),
             "dirz_white_100c60f": dict(n=None, nc=100, nf=60, dir_z=True, white=True, bg=False)}


@pytest.mark.parametrize("case", list(E2E_CASES))
def test_parameter_gradients_against_float64(E, case):
    kw = dict(E2E_CASES[case])
    n = kw.pop("n") or two_iter_rays(E)
    runs = {}
    R = None
    for prec in ("exact", "exact_grad"):
        c = make_case(E, n, kw["nc"], kw["nf"], prec, seed=17, **{k: v for k, v in kw.items() if k not in ("nc", "nf")})
        train_forward(E, c)
        s = saved_state(E, c)
        gouts = out_grads(E, c, seed=5)
        kg = kernel_backward(E, c, gouts)
        if R is None:  # the forward (and so the depths) is the same bits in both modes
            R = reference(E, c, s.z_c, s.z_f, gouts)
        runs[prec] = grad_pairs(kg, R)
    compare(case, runs)


def test_single_ray_gradients_against_float64(E):
    """One ray's output gradients at a time (first, last, and one in the middle of a 2047-ray call)."""
    runs = {"exact": [], "exact_grad": []}
    for prec in runs:
        c = make_case(E, 2047, 64, 64, prec, seed=2)
        train_forward(E, c)
        s = saved_state(E, c)
        dense = out_grads(E, c, seed=3)
        for i in (0, 1000, c.n - 1):
            gouts = []
            for t in dense:
                z = torch.zeros_like(t)
                z[i] = t[i] * c.n
                gouts.append(z)
            kg = kernel_backward(E, c, gouts)
            R = reference(E, c, s.z_c, s.z_f, gouts, lo=i, hi=i + 1)
            runs[prec] += [(f"ray {i} {nm}", g, r) for nm, g, r in grad_pairs(kg, R)]
    compare("single rays", runs)


def test_chunked_gradients_against_float64(E, monkeypatch):
    """Over the memory budget: the backward re-runs the exact-grad training forward chunk by chunk (2 MiB records)."""
    runs = {}
    R = None
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "200")
    for prec in ("exact", "exact_grad"):
        c = make_case(E, 1024, 64, 64, prec, seed=23)
        out = train_forward(E, c)
        torch.cuda.synchronize()
        gouts = out_grads(E, c, seed=5)
        kg = kernel_backward(E, c, gouts)
        if R is None:  # the depths of the evaluation forward: rebuild them from a one-launch forward with the budget lifted
            monkeypatch.setenv("NFB_TRAIN_MEM_MB", "60000")
            train_forward(E, c)
            s = saved_state(E, c)
            monkeypatch.setenv("NFB_TRAIN_MEM_MB", "200")
            R = reference(E, c, s.z_c, s.z_f, gouts)
            del out
        runs[prec] = grad_pairs(kg, R)
    compare("chunked", runs)


def test_input_only_gradients_against_float64(E):
    """Input-only backward (no parameter gradient): the latent through the PE-only weight-gradient launch."""
    runs = {}
    R = None
    for prec in ("exact", "exact_grad"):
        c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=29)
        train_forward(E, c)
        s = saved_state(E, c)
        gouts = out_grads(E, c, seed=5)
        pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
        pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER]
        _, _, gl, _ = E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["background"])
        torch.cuda.synchronize()
        if R is None:
            R = reference(E, c, s.z_c, s.z_f, gouts)
        runs[prec] = [("latent", gl, R.glat)]
    compare("input-only latent", runs)


def test_input_and_expression_gradients_against_float64(E):
    """Per-ray input gradients (origins, directions, dir_z, background; the row and ray kernels) and d expression end to end,
    against tests/test_input_grads_gpu.reference_inputs in float64."""
    from test_input_grads_gpu import input_pairs, kernel_inputs, reference_inputs
    runs = {}
    ref = None
    for prec in ("exact", "exact_grad"):
        c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=43, dir_z=True)
        train_forward(E, c)
        s = saved_state(E, c)
        gouts = out_grads(E, c, seed=5)
        kg, ing = kernel_inputs(E, c, gouts)
        if ref is None:
            ref, R = reference_inputs(E, c, s.z_c, s.z_f, gouts)
        runs[prec] = input_pairs(ing, ref) + [("latent", kg[2], R.glat)]
    compare("inputs + expression", runs, IN_E2E_TOL)


def test_multi_frame_gradients_against_float64(E):
    """F = 5 frames in one call: per-frame latent and expression gradients (raysum_x3_kernel, framesum_kernel), the parameter and
    per-ray input gradients, against tests/test_multi_frame_fp64_gpu.reference_multi in float64."""
    from test_input_grads_gpu import params_of
    from test_multi_frame_fp64_gpu import frames, layout, reference_multi, render
    runs = {}
    R = None
    for prec in ("exact", "exact_grad"):
        c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=47, dir_z=True)
        ex, la = frames(E, 5, 0)
        fi = layout("interleave", c.n, 5, 0)
        E.eng.sync_weights(c.mc, c.mf)
        E.eng.set_frames(ex, la)
        render(E, c, True, fi)
        s = saved_state(E, c)
        gouts = out_grads(E, c, seed=5)
        pc, pf = params_of(c)
        gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=True, frames=True,
                                         inputs=["ray_origins", "ray_directions", "dir_z", "background", "expression"])
        torch.cuda.synchronize()
        if R is None:
            R = reference_multi(E, c, fi, ex, la, s.z_c, s.z_f, gouts)
        pairs = [("latents", gl, R.glat), ("expressions", ing["expression"], R.gexp)]
        pairs += [(k, ing[k], R.ins[k]) for k in R.ins]
        pairs += [(f"c/{k}", g, r) for k, g, r in zip(TR.PARAM_ORDER, gc, R.gc) if g is not None]
        pairs += [(f"f/{k}", g, r) for k, g, r in zip(TR.PARAM_ORDER, gf, R.gf) if g is not None]
        runs[prec] = pairs
    compare("multi-frame F=5", runs, MF_E2E_TOL)


# Every path of the backward against float64 at the kernel's OWN forward state: the kernel's d raw (FP32, the same bits in both
# modes: the compositing backward is unchanged), its ReLU masks and its recorded activations (hi + lo), run through the float64
# weights.  This isolates what exact-grad changes (dX chain, weight-gradient GEMMs, row and per-frame sums, their operands) from
# the forward's own error, which reaches d raw through the compositing backward in both modes.  Checked, per category, exact-grad
# within STATE_TOL and RATIO times below exact mode:
#   acc      every block of both networks' accumulators below the raw-output biases (kAcc0 .. kAcc9, b0 .. b8): the full launch
#   pe_only  dW0, dW3a, db0, db3 of an input-only backward (the PE-only launch, dw_x3_kernel<true>)
#   rows     (dp, d v0) of every sample row (row_x3_kernel), from the float64 dY0, dY3, dY6 through the formula of
#            test_input_grads_fp64_gpu.row_formula64
#   raysum   multi-frame: each ray's sums of dY0 | dY3 (raysum_x3_kernel); fsum: those summed per frame
ACC = {  # name: (accumulator offset, rows, cols); nfb_layout.h kAcc*
    "dW0": (0, 256, 64), "dW1": (16384, 256, 256), "dW2": (16384 + 65536, 256, 256), "dW3a": (16384 + 2 * 65536, 256, 64),
    "dW3b": (2 * 16384 + 2 * 65536, 256, 256), "dW4": (2 * 16384 + 3 * 65536, 256, 256), "dW5": (2 * 16384 + 4 * 65536, 256, 256),
    "dM1": (360448, 128, 256), "dWd0dir": (393216, 128, 32), "dSig": (397312, 256, 16), "dW7": (401408, 128, 128),
    "dW8": (417792, 128, 128), "dW9t": (434176, 128, 16)}
ACC_B = 436224  # kAccB: b0..b5 [256] each, then b6..b8 [128] each
BIAS = {L: (ACC_B + 256 * L if L < 6 else ACC_B + 1536 + 128 * (L - 6), 256 if L < 6 else 128) for L in range(9)}
PE_ONLY = ("dW0", "dW3a", "db0", "db3")


def fold64(p):
    W = {k: v.detach().double() for k, v in p.items()}
    m1 = W["layers_dir.0.weight"][:, :256] @ W["fc_feat.weight"]  # [128, 256]
    m2 = W["fc_alpha.weight"] @ W["fc_feat.weight"]              # [1, 256]
    return W, m1, m2


def pad16(t):
    return torch.cat((t, torch.zeros(t.shape[0], 16 - t.shape[1], dtype=t.dtype, device=t.device)), 1)


def mlp_backward64(W, m1, m2, d_raw, X):
    """float64 pre-activation gradients dA[L] and every accumulator block from d raw [rows, 4] and activations X (masks:
    X != 0), in the accumulators' folded parametrisation (nfb_layout.h kAcc*)."""
    m = {L: (X[L] != 0).double() for L in range(9)}
    dA = {8: (d_raw[:, :3] @ W["fc_rgb.weight"]) * m[8]}
    dA[7] = (dA[8] @ W["layers_dir.2.weight"]) * m[7]
    dA[6] = (dA[7] @ W["layers_dir.1.weight"]) * m[6]
    dA[5] = (dA[6] @ m1 + d_raw[:, 3:4] @ m2) * m[5]
    dA[4] = (dA[5] @ W["layers_xyz.5.weight"]) * m[4]
    dA[3] = (dA[4] @ W["layers_xyz.4.weight"]) * m[3]
    dA[2] = (dA[3] @ W["layers_xyz.3.weight"][:, 171:]) * m[2]
    dA[1] = (dA[2] @ W["layers_xyz.2.weight"]) * m[1]
    dA[0] = (dA[1] @ W["layers_xyz.1.weight"]) * m[0]
    out = {"dW0": dA[0].T @ X["pe"], "dW1": dA[1].T @ X[0], "dW2": dA[2].T @ X[1], "dW3a": dA[3].T @ X["pe"],
           "dW3b": dA[3].T @ X[2], "dW4": dA[4].T @ X[3], "dW5": dA[5].T @ X[4], "dM1": dA[6].T @ X[5], "dWd0dir": dA[6].T @ X["ped"],
           "dSig": pad16(X[5].T @ d_raw), "dW7": dA[7].T @ X[6], "dW8": dA[8].T @ X[7], "dW9t": pad16(X[8].T @ d_raw)}
    for L in range(9):
        out[f"db{L}"] = dA[L].sum(0)
    return dA, out


def acc_blocks(acc, names):
    got = {}
    for name in names:
        if name.startswith("db"):
            off, w = BIAS[int(name[2:])]
            got[name] = acc[off:off + w]
        else:
            off, r, cc = ACC[name]
            got[name] = acc[off:off + r * cc].view(r, cc)
    return got


STATE_CASES = {"64c64f": dict(nc=64, nf=64, multi=False), "64c0f": dict(nc=64, nf=0, multi=False),
               "64c64f_F5": dict(nc=64, nf=64, multi=True)}


@pytest.mark.parametrize("case", list(STATE_CASES))
def test_every_backward_path_at_the_kernels_forward_state(E, case):
    from test_input_grads_fp64_gpu import row_formula64
    from test_input_grads_gpu import params_of
    from test_multi_frame_fp64_gpu import frames, layout, render
    kw = STATE_CASES[case]
    nc, nf, multi = kw["nc"], kw["nf"], kw["multi"]
    inputs = ["ray_origins", "ray_directions", "dir_z", "background"]
    errs = {"exact": {}, "exact_grad": {}}
    X = None
    for prec in ("exact_grad", "exact"):
        c = make_case(E, two_iter_rays(E), nc, nf, prec, seed=41, dir_z=True)
        E.eng.sync_weights(c.mc, c.mf)
        if multi:
            ex, la = frames(E, 5, 0)
            fi = layout("interleave", c.n, 5, 0)
            E.eng.set_frames(ex, la)
            render(E, c, True, fi)
        else:
            train_forward(E, c)
        s = saved_state(E, c)
        s.rays = dev_tensor(s.dbg.rays, (c.n, 7)).clone()
        gouts = out_grads(E, c, seed=5)
        pc, pf = params_of(c)
        E.eng.backward(list(gouts), pc, pf, want_params=True, inputs=inputs, frames=multi)
        torch.cuda.synchronize()
        d = E.eng.train_debug()
        tpu, npass = s.tc + s.tf, 2 if nf else 1
        accs = [dev_tensor(d.acc_coarse, (int(d.acc_floats),)).clone()] + ([dev_tensor(d.acc_fine, (int(d.acc_floats),)).clone()] if nf else [])
        rows = dev_tensor(d.rows, (s.n_tiles, 128, 4)).clone()
        if multi:
            raysum = dev_tensor(d.ray_sums, (npass, c.n, 512)).clone()
            fsum = dev_tensor(d.frame_sums, (5, 2, 512)).clone()
            frame = dev_tensor(d.frame, (c.n,), "<i4").clone().long()
        else:  # an input-only backward with d latent: the PE-only weight-gradient launch
            E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["expression"])
            torch.cuda.synchronize()
            d = E.eng.train_debug()
            assert d.dw_pe_only == 1
            pe_accs = [dev_tensor(d.acc_coarse, (int(d.acc_floats),)).clone()] + ([dev_tensor(d.acc_fine, (int(d.acc_floats),)).clone()] if nf else [])
        if X is None:  # the exact-grad records: hi + lo of every activation, and the masks (hi != 0)
            rec = dev_tensor(d.records, (s.n_tiles, 2 * MIB), "|u1").view(torch.int16)
            hi16, lo16 = rec[:, :MIB // 2].contiguous(), rec[:, MIB // 2:].contiguous()
            X = {L: decode_image(hi16, x_off(L), 256 if L < 6 else 128) + decode_image(lo16, x_off(L), 256 if L < 6 else 128)
                 for L in range(9)}
            X["pe"] = decode_image(hi16, 0, 64) + decode_image(lo16, 0, 64)
            X["ped"] = decode_image(hi16, PED_OFF, 32) + decode_image(lo16, PED_OFF, 32)
            d_raw = dev_tensor(d.d_raw, (s.n_tiles, 128, 4)).clone()
            del rec, hi16, lo16
        else:
            assert torch.equal(d_raw, dev_tensor(d.d_raw, (s.n_tiles, 128, 4)))  # d raw: the same bits in both modes
        e = errs[prec]
        ray_db = torch.zeros(npass, c.n, 512, dtype=torch.float64, device=E.dev)
        for net, model in enumerate([c.mc] + ([c.mf] if nf else [])):
            tiles = torch.tensor([t for t in range(s.n_tiles) if ((t % tpu) >= s.tc) == bool(net)], device=E.dev)
            pos = torch.full((s.n_tiles,), -1, dtype=torch.long, device=E.dev)
            pos[tiles] = torch.arange(len(tiles), device=E.dev)
            Xn = {k: v[tiles].reshape(-1, v.shape[-1]).double() for k, v in X.items()}
            dA, ref = mlp_backward64(*fold64(dict(model.named_parameters())), d_raw[tiles].reshape(-1, 4).double(), Xn)
            got = acc_blocks(accs[net].double(), ref)
            e.setdefault("acc", []).extend((f"{net}/{k}", got[k], ref[k]) for k in ref)
            if not multi:
                got = acc_blocks(pe_accs[net].double(), PE_ONLY)
                e.setdefault("pe_only", []).extend((f"{net}/{k}", got[k], ref[k]) for k in PE_ONLY)
            tile, row = rowmap(c, s, net)
            S = c.nc + c.nf if net else c.nc
            at = pos[tile] * 128 + row
            ray = torch.arange(tile.numel(), device=E.dev) // S
            z = (s.z_f if net else s.z_c).reshape(-1)
            rref, _ = row_formula64(c, s, model, 1.0, dA[0][at], dA[3][at], dA[6][at], ray, z)
            e.setdefault("rows", []).append((f"{net}/rows", rows[tile, row], rref))
            ray_db[net] = torch.cat((dA[0][at], dA[3][at]), 1).view(c.n, S, 512).sum(1)
        if multi:
            e["raysum"] = [(f"{p}/raysum", raysum[p], ray_db[p]) for p in range(npass)]
            fref = torch.zeros(5, 2, 512, dtype=torch.float64, device=E.dev)
            for p in range(npass):
                fref[:, p].index_add_(0, frame, ray_db[p])
            e["fsum"] = [("fsum", fsum, fref)]
    for cat in errs["exact_grad"]:
        (xm, xl), (gm, gl) = worst(errs["exact"][cat]), worst(errs["exact_grad"][cat])
        print(f"kernel state {case} {cat}: exact max {xm:.2e} L2 {xl:.2e}; exact_grad max {gm:.2e} L2 {gl:.2e}; "
              f"ratio {xm / gm:.0f}x, {xl / gl:.0f}x")
        assert gm <= STATE_TOL[0] and gl <= STATE_TOL[1], (case, cat, gm, gl)
        assert gm * RATIO <= xm and gl * RATIO <= xl, (case, cat, xm, gm, xl, gl)


# ---------------------------------------------------------------------------------------------------------------- (d)
def test_backward_repeats_bit_for_bit(E):
    c = make_case(E, two_iter_rays(E), 64, 128, "exact_grad", seed=31)
    gouts = out_grads(E, c, seed=5)
    train_forward(E, c)
    a = kernel_backward(E, c, gouts)
    b = kernel_backward(E, c, gouts)  # the same saved forward again
    train_forward(E, c)
    d = kernel_backward(E, c, gouts)  # a second run from the forward
    for x, y, z in zip(*[[t for t in list(k[0]) + list(k[1]) + [k[2]] if t is not None] for k in (a, b, d)]):
        assert torch.equal(x, y) and torch.equal(x, z)


@pytest.mark.parametrize("what", ["nan_input", "fp16_overflow"])
def test_non_finite_gradients(E, what):
    """A NaN ray direction, or a hidden activation beyond the FP16 range (an input scaled up), gives non-finite gradients."""
    c = make_case(E, two_iter_rays(E), 64, 64, "exact_grad", seed=37)
    if what == "nan_input":
        c.rd = c.rd.clone()
        c.rd[5, 1] = float("nan")
    else:
        sd = {k: v.detach().clone() for k, v in c.mc.state_dict().items()}
        sd["layers_xyz.1.weight"] *= 4000.0
        from test_backward_fp64_gpu import model
        c.mc = model(E, 0, True, params={k: v.cpu() for k, v in sd.items()})
    train_forward(E, c)
    gc, gf, gl = kernel_backward(E, c, out_grads(E, c, seed=5))
    assert not all(bool(torch.isfinite(t).all()) for t in list(gc) + [gl] if t is not None), what


def test_precision_three_is_invalid(E):
    c = make_case(E, 8, 64, 64, "exact", seed=1)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    sm = E.eng._sampling(64, 64, "exact", False)
    sm.precision = 3
    out = {k: torch.zeros(8, 3 if k.startswith("rgb") else 1, device=E.dev) for k in NAMES}
    rays = E.capi.NfbRays()
    rays.o, rays.d, rays.n_rays, rays.near_, rays.far_ = c.ro.data_ptr(), c.rd.data_ptr(), 8, 0.2, 0.8
    outs = E.capi.NfbOutputs(*[out[k].data_ptr() for k in NAMES])
    lib, h = E.capi.lib, E.eng._h
    for prec, want in ((3, 1), (-1, 1), (2, 0)):  # NFB_ERR_INVALID outside 0..2; exact-grad itself renders
        sm.precision = prec
        assert lib.nfb_render_forward(h, C.byref(rays), C.byref(sm), None, C.byref(outs), None, None) == want, prec
        assert lib.nfb_render_forward_train(h, C.byref(rays), C.byref(sm), None, C.byref(outs), None) == want, prec
    E.eng.set_frames(c.expr.reshape(1, 76), c.latent.reshape(1, 32))
    fi = torch.zeros(8, dtype=torch.int32, device=E.dev)
    sm.precision = 3
    assert lib.nfb_render_forward_frames(h, C.byref(rays), C.c_void_p(fi.data_ptr()), C.byref(sm), None, C.byref(outs), None) == 1
    assert lib.nfb_render_forward_frames_train(h, C.byref(rays), C.c_void_p(fi.data_ptr()), C.byref(sm), None, C.byref(outs),
                                               None) == 1
    pose = (C.c_float * 12)(*[1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0])
    intr = (C.c_double * 4)(8.0, 8.0, 0.5, 0.5)
    host = torch.zeros(11 * 16)
    e_h, l_h = c.expr.cpu().contiguous(), c.latent.cpu().contiguous()
    assert lib.nfb_render_frame_host(h, pose, intr, 4, 4, 0, 4, C.c_float(0.2), C.c_float(0.8), C.c_void_p(e_h.data_ptr()),
                                     C.c_void_p(l_h.data_ptr()), None, C.byref(sm), C.c_void_p(host.data_ptr()), None) == 1
    with pytest.raises(ValueError):  # the Python surface refuses a misspelt mode rather than rendering in fast mode
        E.eng.render(c.ro, c.rd, 0.2, 0.8, 64, 64, precision="exact-grad")
