"""The input-gradient path of nfb_render_backward_ex (csrc/nfb_train.cu) against float64, stage by stage, at every tile of
the row kernel's schedule, and at its routing, FP16-range, loss-scale and non-finite edges.

The path has four stages after the compositing backward and the dX chain; each is fed the kernel's own output of the stage
before it, read through NfbTrainDebug (rays, dnorm, rows, ray_dn, ray_bg, records, accumulators):
  (a) saved rays     (o, d) bitwise the caller's; v0 bitwise dir_z (d_z without one); |d| bitwise the forward's FP32 formula
                     sqrt((d0 d0 + d1 d1) + d2 d2).
  (b) compositing    ray_dn [pass][ray] = dL/d|d| and ray_bg [pass][ray][3] = dL/d background against float64 autograd of the
                     compositing alone, at the kernel's saved sigma inputs, colours and depths, |d| and the background as
                     leaves: max-abs / max|ref| and relative L2 over the rays of each pass, COMP_TOL.
  (c) rows           every live row's (dp, d v0) against float64 of the formula above ing::row_kernel, from the decoded dY0,
                     dY3, dY6 records times scale[1], the FP32 master columns, v0 from `rays` and the point o + d z formed in
                     FP32 as the forward forms it (two roundings), then promoted.  Per row and component the error is bounded
                     relative to the same sum over absolute values (|W|^T |dY|, |sin|, |cos|), ROW_TOL.  Rows that hold no
                     sample are exactly 0.  The per-row error is uniform (KAPPA, test_render_fp64_gpu.check_uniformity) over
                     the row kernel's schedule classes: network x CTA part (tile j mod parts), and network x CTA iteration
                     (j / parts: 0 or >= 1) x tile within the unit x warp (row / 32).  With more than 3 rays, the float64
                     formula at the once-rounded point fma(d, z, o) must differ from the twice-rounded one by more than
                     ROW_TOL: the bound resolves a one-ulp change of the point, so a row kernel forming p with fmaf fails.
  (d) rays           d o, d d, d dir_z (or d_z) and d bg against float64 sums of the kernel's own rows over both passes
                     with z, ray_dn, ray_bg, dnorm and rays, relative to the sums of absolute values, RAY_TOL.
  (e) conditioning   d expression and d latent against float64 from the kernel's own layer-0 / layer-3 bias sums in the
                     accumulators, in input-only mode (cond_grad_kernel) and in full mode (finalize_kernel), COND_TOL.
  (f) end to end     against test_input_grads_gpu.reference_inputs at its bounds (IN_TOL).

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases and both modes:
  (b) max 4.9e-6, L2 3.4e-6 (256c+256f)                                           -> COMP_TOL (2e-5, 1e-5)
  (c) rows 1.4e-7 of the absolute sum                                              -> ROW_TOL 5e-7
      the fma(d, z, o) reference against the o + d z one: 1.6e-6 to 3.2e-6 with more than 3 rays (1.2e-6 with 1-3)
      worst class RMS / overall RMS: 1.28                                          -> KAPPA 2.5
  (d) 1.6e-7 of the absolute sum                                                   -> RAY_TOL 1e-6
  (e) 1.4e-7 of the absolute sum                                                   -> COND_TOL 1e-6
  (f) within IN_TOL (with 1-3 rays the single-ray PROBE_TOL; 3c+0f fast's latent the TOL_3C_FAST of test_backward_fp64_gpu);
      origins moved by 50 (random-init weights): exact max 2.3e-2, L2 1.0e-2 -> PROBE_TOL, see run_stages
  non-finite edges: at least 99.6 % of the parameter-gradient entries float64 makes non-finite are non-finite in the kernel
                                                                                   -> NONFIN_SHARE 0.9
Defects these tests were checked against, each built once, each failing the stage check named: the sin and cos direction
columns swapped in row_kernel (rows, 0.36-0.50 of the absolute sum), row_kernel skipping PE column 62 (rows, 0.14),
row_kernel reading network 0's weights on fine tiles (rows of the fine pass, 0.45), ray_kernel dropping the fine pass's |d|
term (d ray_directions, 1.7e-2); p formed with one rounding (fmaf) in row_kernel: rows 2.0e-6 to 2.6e-6 at origins
within 1, 9.6e-5 at origins moved by 50.  Before the compositing
backward kept NaN, a NaN sigma-noise draw with fixed output gradients gave finite gradients (test_nonfinite_inputs).
"""
import ctypes as C
import types

import pytest
import torch

import torch_reference as TR
from test_backward_gpu import decode_image, dev_tensor, dy_off
from test_backward_fp64_gpu import (E, PROBE_TOL, TOL, TOL_3C_FAST, check, grad_pairs, make_case, model, out_grads,  # noqa: F401
                                    reference, rowmap, saved_state, train_forward, two_iter_rays)
from test_input_grads_gpu import IN_TOL, input_pairs, params_of, reference_inputs, wanted
from test_render_fp64_gpu import check_uniformity

pytestmark = pytest.mark.gpu

PRECS = ["exact", "fast"]
COMP_TOL = (2e-5, 1e-5)     # (max-abs / max|ref|, relative L2) of ray_dn and ray_bg per pass
ROW_TOL = 5e-7              # |row - ref| / (sum of absolute values), per row and component
RAY_TOL = 1e-6              # per-ray sums, relative to the sums of absolute values
COND_TOL = 1e-6             # d expression, d latent, relative to the sums of absolute values
ACC_FLOATS = 438148         # nfb_layout.h kAccFloats
ACC_B = 436224              # nfb_layout.h kAccB: the layer biases, 256 floats each for layers 0..5
RAY_INPUTS = ("ray_origins", "ray_directions", "dir_z", "background")
NONFIN_SHARE = 0.9          # parameter-gradient entries float64 makes non-finite that must be non-finite in the kernel


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def debug_state(E, c):
    """saved_state plus the saved rays and |d| of the last (one-launch) training forward."""
    s = saved_state(E, c)
    s.rays = dev_tensor(s.dbg.rays, (c.n, 7)).clone()
    s.dnorm = dev_tensor(s.dbg.dnorm, (c.n,)).clone()
    s.raw = [dev_tensor(s.dbg.raw_coarse, (c.n, c.nc, 4)).clone()]
    if c.nf:
        s.raw.append(dev_tensor(s.dbg.raw_fine, (c.n, c.nc + c.nf, 4)).clone())
    return s


def backward_state(E, c, s, gouts, want_params=False, inputs=None):
    """One backward with input gradients; returns its results and what it left in the training state."""
    pc, pf = params_of(c)
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=want_params,
                                     inputs=list(wanted(c) if inputs is None else inputs))
    torch.cuda.synchronize()
    d = E.eng.train_debug()
    npass = 2 if c.nf else 1
    assert d.acc_floats == ACC_FLOATS
    t = types.SimpleNamespace(kg=(gc, gf, gl), ing=ing, dbg=d)
    t.rows = dev_tensor(d.rows, (s.n_tiles, 128, 4)).clone() if d.rows else None
    t.ray_dn = dev_tensor(d.ray_dn, (npass, c.n)).clone() if d.ray_dn else None
    t.ray_bg = dev_tensor(d.ray_bg, (npass, c.n, 3)).clone() if d.ray_bg else None
    t.inv = float(dev_tensor(d.scale, (2,))[1])
    t.acc = [dev_tensor(d.acc_coarse, (ACC_FLOATS,)).clone()] + ([dev_tensor(d.acc_fine, (ACC_FLOATS,)).clone()] if c.nf else [])
    return t


def bounded(tag, got, ref, bound, tol):
    """max over entries of |got - ref| / bound (an entry whose bound is 0 must be met exactly)."""
    diff = (got.double() - ref).abs()
    r = torch.where(bound > 0, diff / bound.clamp(min=1e-300), torch.where(diff > 0, float("inf"), 0.0))
    worst = float(r.max()) if r.numel() else 0.0
    assert worst <= tol, (tag, worst)
    return worst, r


# ---------------------------------------------------------------------------------------------------------------- (a)
def check_saved_rays(c, s, tag):
    ro, rd, rays = c.ro.cpu(), c.rd.cpu(), s.rays.cpu()
    assert same_bits(rays[:, 0:3], ro) and same_bits(rays[:, 3:6], rd), (tag, "saved o, d")
    v0 = c.dz.cpu() if c.dz is not None else rd[:, 2]
    assert same_bits(rays[:, 6], v0), (tag, "saved v0")
    # IEEE FP32 with one rounding per operation, emulated in float64 (exact products and sums, then one rounding; the square
    # root rounded twice is still the FP32 one).  torch's own FP32 sqrt on the CPU is not correctly rounded.
    r32 = lambda x: x.float().double()  # noqa: E731
    d = rd.double()
    dn = r32(torch.sqrt(r32(r32(r32(d[:, 0] * d[:, 0]) + r32(d[:, 1] * d[:, 1])) + r32(d[:, 2] * d[:, 2])))).float()
    assert same_bits(s.dnorm.cpu(), dn), (tag, "saved |d|", int((bits(s.dnorm.cpu()) != bits(dn)).sum()))


# ---------------------------------------------------------------------------------------------------------------- (b)
def composite_terms64(c, s, pas, gouts):
    """float64 dL/d|d|, dL/d background and d raw [n, S, 4] = (dL/d rgb_raw, dL/d sigma_raw) of one pass's compositing, at
    the kernel's saved sigma inputs, colours, depths: d rgb_raw = dL/dc c (1 - c) from the saved colour c, d sigma_raw through
    the ReLU of the saved input."""
    z = (s.z_f if pas else s.z_c).double()
    raw = s.raw[pas].double().requires_grad_(True)
    dn = s.dnorm.double().requires_grad_(True)
    bg = c.bg.double().requires_grad_(True) if c.bg is not None else None
    col = raw[..., :3] if bg is None else torch.cat((raw[:, :-1, :3], bg[:, None, :]), dim=1)
    last = torch.zeros(z.shape[1], dtype=torch.float64, device=z.device)
    last[-1] = 1e-6
    sigma = torch.relu(raw[..., 3]) + last
    delta = torch.cat((z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)), dim=-1) * dn[:, None]
    alpha = 1.0 - torch.exp(-sigma * delta)
    trans = torch.cumprod(1.0 - alpha + 1e-10, dim=-1)
    w = alpha * torch.cat((torch.ones_like(trans[:, :1]), trans[:, :-1]), dim=-1)
    rgb = (w[..., None] * col).sum(dim=-2)
    depth, acc = (w * z).sum(dim=-1), w.sum(dim=-1)
    disp = 1.0 / torch.max(1e-10 * torch.ones_like(depth), depth / acc)
    if c.white:
        rgb = rgb + (1.0 - acc[..., None])
    outs = [(rgb, gouts[3 * pas]), (disp, gouts[3 * pas + 1]), (acc, gouts[3 * pas + 2])]
    if pas == (1 if c.nf else 0):
        outs.append((w[:, -1], gouts[6]))
    loss = sum((o * g.double()).sum() for o, g in outs if g is not None)
    loss.backward()
    col = raw.detach()[..., :3]
    d_raw = torch.cat((raw.grad[..., :3] * col * (1.0 - col), raw.grad[..., 3:]), dim=-1)
    return dn.grad, (bg.grad if bg is not None else None), d_raw


def check_compositing_terms(c, s, t, gouts, tag):
    worst = [0.0, 0.0]
    for pas in range(2 if c.nf else 1):
        gdn, gbg, _ = composite_terms64(c, s, pas, gouts)
        pairs = [("ray_dn", t.ray_dn[pas], gdn)] + ([("ray_bg", t.ray_bg[pas], gbg)] if gbg is not None else [])
        for name, got, ref in pairs:
            assert bool(torch.isfinite(got).all()), (tag, pas, name)
            d = (got.double() - ref).abs()
            rmax = float(ref.abs().max())
            em = float(d.max()) / rmax if rmax > 0 else (0.0 if float(d.max()) == 0 else float("inf"))
            el = float(d.norm() / ref.norm()) if rmax > 0 else em
            worst = [max(worst[0], em), max(worst[1], el)]
            assert em <= COMP_TOL[0] and el <= COMP_TOL[1], (tag, pas, name, em, el)
    assert (t.ray_bg is None) == (c.bg is None), tag
    return worst


# ---------------------------------------------------------------------------------------------------------------- (c)
def row_parts(E, c, s):
    """The row kernel's CTA split: dw_split(num_sms * 8 job groups, tiles of each network), as launch_input_grads calls it."""
    n_units = (c.n + s.R - 1) // s.R
    buf = (C.c_uint32 * 16)(E.sms * 8, n_units * s.tc, n_units * s.tf if c.nf else 0)
    assert E.capi.lib.nfb_debug_schedule(4, 0, buf, 16) == 3
    return int(buf[0]), int(buf[1])


def row_formula64(c, s, m, inv, dy0, dy3, dy6, ray, z, fused=False):
    """float64 (dp, d v0) and the same sum over absolute values, for rows of one network (the comment above ing::row_kernel)."""
    P = dict(m.named_parameters())
    W0 = P["layers_xyz.0.weight"].detach().double()[:, :63]
    W3 = P["layers_xyz.3.weight"].detach().double()[:, :63]
    Wd = P["layers_dir.0.weight"].detach().double()[:, 256:280]
    g0, g3, g6 = dy0.double() * inv, dy3.double() * inv, dy6.double() * inv
    dpe = g0 @ W0 + g3 @ W3
    ape = g0.abs() @ W0.abs() + g3.abs() @ W3.abs()
    dpd, apd = g6 @ Wd, g6.abs() @ Wd.abs()
    o, d = s.rays[ray, 0:3], s.rays[ray, 3:6]
    if fused:  # one rounding: d z is exact in float64
        p = (o.double() + d.double() * z.double()[:, None]).float().double()
    else:      # as the forward: fl(o + fl(d z))
        p = (o + d * z[:, None]).double()
    N = p.shape[0]
    f = (2.0 ** torch.arange(10, dtype=torch.float64, device=p.device)).view(1, 10, 1)
    x = p[:, None, :] * f
    cs, sn = torch.cos(x), torch.sin(x)
    hs, hc = dpe[:, 3:].view(N, 10, 6)[:, :, :3], dpe[:, 3:].view(N, 10, 6)[:, :, 3:]
    As, Ac = ape[:, 3:].view(N, 10, 6)[:, :, :3], ape[:, 3:].view(N, 10, 6)[:, :, 3:]
    dp = dpe[:, :3] + (f * (cs * hs - sn * hc)).sum(1)
    ap = ape[:, :3] + (f * (cs.abs() * As + sn.abs() * Ac)).sum(1)
    v0 = s.rays[ray, 6].double()
    fd = 2.0 ** torch.arange(4, dtype=torch.float64, device=p.device)
    xd = v0[:, None] * fd
    ds, dc = dpd.view(N, 4, 6)[:, :, 0], dpd.view(N, 4, 6)[:, :, 3]
    As_, Ac_ = apd.view(N, 4, 6)[:, :, 0], apd.view(N, 4, 6)[:, :, 3]
    dv = (fd * (torch.cos(xd) * ds - torch.sin(xd) * dc)).sum(1)
    av = (fd * (torch.cos(xd).abs() * As_ + torch.sin(xd).abs() * Ac_)).sum(1)
    return torch.cat((dp, dv[:, None]), 1), torch.cat((ap, av[:, None]), 1)


def check_rows(E, c, s, t, tag, chunk=1 << 16, dy=None):
    """dy: the decoded dY0, dY3, dY6 images the row kernel read (by default the FP16 records; exact-grad passes hi + lo)."""
    if dy is None:
        recs = dev_tensor(t.dbg.records, (s.n_tiles, t.dbg.record_bytes // 2), "<i2")
        dy = [decode_image(recs, dy_off(L), 256 if L < 6 else 128) for L in (0, 3, 6)]
    used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=E.dev)
    parts = row_parts(E, c, s)
    tpu = s.tc + s.tf
    worst, fused_gap = 0.0, 0.0
    errs, cls_part, cls_joint = [], [], []
    for pas in range(2 if c.nf else 1):
        tile, row = rowmap(c, s, pas)
        used[tile, row] = True
        S = c.nc + c.nf if pas else c.nc
        z = (s.z_f if pas else s.z_c).reshape(-1)
        m = c.mf if pas else c.mc
        for b in range(0, tile.numel(), chunk):
            e = min(tile.numel(), b + chunk)
            tl, rw = tile[b:e], row[b:e]
            ray = torch.arange(b, e, device=E.dev) // S
            args = (c, s, m, t.inv, dy[0][tl, rw], dy[1][tl, rw], dy[2][tl, rw], ray, z[b:e])
            ref, bound = row_formula64(*args)
            w, r = bounded(f"{tag} rows pass {pas}", t.rows[tl, rw], ref, bound, ROW_TOL)
            worst = max(worst, w)
            fref, _ = row_formula64(*args, fused=True)
            fused_gap = max(fused_gap, float(((fref - ref).abs() / bound.clamp(min=1e-300)).max()))
            errs.append(r.max(1).values.pow(2))
            j = (tl // tpu) * (s.tf if pas else s.tc) + (tl % tpu) - (s.tc if pas else 0)
            P = parts[pas]
            cls_part.append(pas * 4096 + j % P)
            cls_joint.append((((pas * 2 + (j // P).clamp(max=1)) * 8 + (tl % tpu)) * 4 + rw // 32))
    if bool((~used).any()):
        assert float(t.rows[~used].abs().max()) == 0.0, (tag, "a row without a sample")
    errs = torch.cat(errs)
    k1 = check_uniformity(f"{tag} rows by CTA part", errs, torch.cat(cls_part))
    k2 = check_uniformity(f"{tag} rows by iteration x tile x warp", errs, torch.cat(cls_joint))
    if c.n > 3:  # the bound resolves a one-ulp change of the point: a row kernel forming p with fmaf fails it
        assert fused_gap > ROW_TOL, (tag, fused_gap)
    return worst, max(k1, k2), fused_gap


# ---------------------------------------------------------------------------------------------------------------- (d)
def check_rays(c, s, t, tag):
    n = c.n
    rows = t.rows.double()
    so, ao = torch.zeros(n, 3, dtype=torch.float64, device=rows.device), torch.zeros(n, 3, dtype=torch.float64, device=rows.device)
    sd, ad = torch.zeros_like(so), torch.zeros_like(so)
    sv, av = torch.zeros(n, dtype=torch.float64, device=rows.device), torch.zeros(n, dtype=torch.float64, device=rows.device)
    for pas in range(2 if c.nf else 1):
        tile, row = rowmap(c, s, pas)
        S = c.nc + c.nf if pas else c.nc
        r = rows[tile, row].view(n, S, 4)
        z = (s.z_f if pas else s.z_c).double()[..., None]
        so += r[..., :3].sum(1)
        ao += r[..., :3].abs().sum(1)
        sd += (z * r[..., :3]).sum(1)
        ad += (z * r[..., :3]).abs().sum(1)
        sv += r[..., 3].sum(1)
        av += r[..., 3].abs().sum(1)
    dn, d = s.dnorm.double(), s.rays[:, 3:6].double()
    sd += (t.ray_dn.double().sum(0) / dn)[:, None] * d
    ad += (t.ray_dn.double().abs().sum(0) / dn)[:, None] * d.abs()
    ref = {"ray_origins": (so, ao), "ray_directions": (sd, ad)}
    if c.dz is not None:
        ref["dir_z"] = (sv, av)
    else:
        sd[:, 2] += sv
        ad[:, 2] += av
    if c.bg is not None:
        ref["background"] = (t.ray_bg.double().sum(0), t.ray_bg.double().abs().sum(0))
    worst = 0.0
    for name, (r, a) in ref.items():
        worst = max(worst, bounded(f"{tag} {name}", t.ing[name], r, a, RAY_TOL)[0])
    return worst


# ---------------------------------------------------------------------------------------------------------------- (e)
def check_cond(c, t, tag):
    se = torch.zeros(76, dtype=torch.float64, device=t.acc[0].device)
    ae, sl, al = torch.zeros_like(se), torch.zeros(32, dtype=torch.float64, device=se.device), torch.zeros(32, dtype=torch.float64, device=se.device)
    for net, m in enumerate([c.mc] + ([c.mf] if c.nf else [])):
        P = dict(m.named_parameters())
        W0, W3 = P["layers_xyz.0.weight"].detach().double(), P["layers_xyz.3.weight"].detach().double()
        b0 = t.acc[net][ACC_B:ACC_B + 256].double()
        b3 = t.acc[net][ACC_B + 3 * 256:ACC_B + 4 * 256].double()
        for W, b in ((W0, b0), (W3, b3)):
            se += W[:, 63:139].t() @ b
            ae += W[:, 63:139].abs().t() @ b.abs()
            sl += W[:, 139:171].t() @ b
            al += W[:, 139:171].abs().t() @ b.abs()
    w1 = bounded(f"{tag} expression", t.ing["expression"], se / 3.0, ae / 3.0, COND_TOL)[0]
    w2 = bounded(f"{tag} latent", t.kg[2], sl, al, COND_TOL)[0]
    return max(w1, w2)


# ---------------------------------------------------------------------------------------------------------------- cases
def run_stages(E, c, tag, far=False):
    train_forward(E, c)
    s = debug_state(E, c)
    check_saved_rays(c, s, tag)
    gouts = out_grads(E, c)
    t = backward_state(E, c, s, gouts)                      # input-only mode: cond_grad_kernel
    comp = check_compositing_terms(c, s, t, gouts, tag)
    rw, kappa, gap = check_rows(E, c, s, t, tag)
    ry = check_rays(c, s, t, tag)
    cond = check_cond(c, t, tag + " input-only")
    tf = backward_state(E, c, s, gouts, want_params=True)   # full mode: finalize_kernel
    cond = max(cond, check_cond(c, tf, tag + " full"))
    for k in t.ing:
        assert torch.equal(t.ing[k], tf.ing[k]) or k == "expression", (tag, k, "input-only and full backward differ")
    ref, R = reference_inputs(E, c, s.z_c, s.z_f, gouts)
    # With 1-3 rays every tensor is a per-ray comparison: the single-ray bounds of the scheduling probes apply.  At origins
    # moved by 50 the float64 reference evaluates the network at o + d z without the FP32 rounding of the point, one ulp of
    # which is 1e-3 rad at frequency 2^9; the forward differs from it by that much, so the single-ray bounds apply there too
    # (stages (a)-(e) are fed the kernel's own FP32 points and keep their bounds).
    tol = IN_TOL[c.prec] if c.n > 3 and not far else PROBE_TOL[c.prec]
    e2e = check(f"{tag} end to end", input_pairs(t.ing, ref), tol, quiet=True)
    check(f"{tag} latent", [("latent", t.kg[2], R.glat)], TOL_3C_FAST if (c.nc, c.prec) == (3, "fast") else TOL[c.prec], quiet=True)
    print(f"{tag}: compositing max {comp[0]:.1e} L2 {comp[1]:.1e}; rows {rw:.1e} (class RMS / overall {kappa:.2f}; "
          f"fma(d, z, o) reference {gap:.1e}); rays {ry:.1e}; conditioning {cond:.1e}; end to end max {e2e[0]:.1e} L2 {e2e[1]:.1e}")


def _prod(stress):
    return lambda E, prec: make_case(E, 2048, 64, 64, prec, stress=stress, seed=50)


def _counts(nc, nf):
    return lambda E, prec: make_case(E, two_iter_rays(E), nc, nf, prec, seed=nc + nf)


def _opt(seed=7, **kw):
    return lambda E, prec: make_case(E, two_iter_rays(E), 64, 64, prec, seed=seed, **kw)


def _far(E, prec):
    """Origins moved by about 50, depths unchanged: p carries 2^-18 ulps, and 2^9 p turns one ulp into 2e-3 rad.
    Random-init weights, so that the gradient reaches most samples of a ray."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, stress=False, seed=9, dir_z=True)
    c.ro = (c.ro + torch.tensor([30.0, -28.0, 29.0], device=E.dev)).contiguous()
    return c


CASES = {
    "prod2048_random_init": _prod(False),
    "prod2048_stress": _prod(True),
    # 4 * SMs + 37 rays: every CTA of the forward and the chain runs two units; the last unit is half filled
    "64c64f": _counts(64, 64),
    "100c60f": _counts(100, 60),       # rays straddle tiles
    "40c24f": _counts(40, 24),
    "256c256f": _counts(256, 256),     # one ray per unit; 16 samples per lane in ray_kernel
    "64c0f": _counts(64, 0),
    "3c0f": _counts(3, 0),
    "white_nobg": _opt(seed=3, white=True, bg=False),   # (the cases of test_input_grads_gpu.test_compositing_options)
    "nobg": _opt(seed=3, bg=False),
    "dir_z": _opt(dir_z=True),
    "deterministic": _opt(perturb=False, noise_std=0.0),
    "1ray": lambda E, prec: make_case(E, 1, 64, 64, prec, seed=1),
    "2rays": lambda E, prec: make_case(E, 2, 64, 64, prec, seed=2),
    "3rays": lambda E, prec: make_case(E, 3, 64, 64, prec, seed=3),
    "far_origin": _far,
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(CASES))
def test_input_grad_stages_against_float64(E, case, prec):
    run_stages(E, CASES[case](E, prec), f"{case} {prec}", far=case == "far_origin")


def test_debug_hook_fields(E):
    """rows / ray_dn / ray_bg stay NULL until a one-launch backward has formed them; a chunked state is NFB_ERR_STATE."""
    c = make_case(E, 300, 64, 64, "fast", seed=5)
    train_forward(E, c)
    s = debug_state(E, c)
    d = E.eng.train_debug()
    assert d.rays and d.dnorm and not d.rows and not d.ray_dn and not d.ray_bg
    gouts = out_grads(E, c)
    t = backward_state(E, c, s, gouts, want_params=True, inputs=[])
    assert t.rows is None and t.ray_dn is None and t.ray_bg is None
    t = backward_state(E, c, s, gouts, inputs=["background"])
    assert t.rows is None and t.ray_dn is not None and t.ray_bg is not None
    t = backward_state(E, c, s, gouts)
    assert t.rows is not None and t.ray_dn is not None and t.ray_bg is not None
    train_forward(E, c)
    d = E.eng.train_debug()
    assert not d.rows and not d.ray_dn and not d.ray_bg


# ---------------------------------------------------------------------------------------------------------------- routing
def one_ray(c, i):
    d = types.SimpleNamespace(**vars(c))
    sl = slice(i, i + 1)
    d.n, d.ro, d.rd = 1, c.ro[sl], c.rd[sl]
    d.bg = c.bg[sl] if c.bg is not None else None
    d.dz = c.dz[sl] if c.dz is not None else None
    d.noise = {k: v[sl] for k, v in c.noise.items()}
    return d


def ray_reference(E, c, s, gouts, i):
    sl = slice(i, i + 1)
    return reference_inputs(E, one_ray(c, i), s.z_c[sl], s.z_f[sl] if c.nf else None,
                            [g[sl] if g is not None else None for g in gouts])


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("nc,nf", [(64, 64), (100, 60)], ids=["64c64f", "100c60f"])
def test_routing_probes(E, nc, nf, prec):
    """2047 rays, one training forward, then per probe ray a backward with output gradients on that ray only.  Probes: the
    rays of the row kernel's first and second CTA iterations (first and last CTA of each network), every ray of the first,
    a middle and the last unit (at 100c+60f their rows straddle tiles).  The probe's input gradients match float64 for that
    ray; every other ray's origin, direction, dir_z and background gradients are exactly 0 (their d raw and dY rows are)."""
    c = make_case(E, 2047, nc, nf, prec, seed=60, dir_z=True)
    train_forward(E, c)
    s = debug_state(E, c)
    n_units = (c.n + s.R - 1) // s.R
    probes = set()
    for pas, P in enumerate(row_parts(E, c, s)):
        S, t_cnt = (c.nc + c.nf, s.tf) if pas else (c.nc, s.tc)
        for j in (0, P - 1, P, 2 * P - 1):
            if 0 <= j < n_units * t_cnt:
                unit, tl = divmod(j, t_cnt)
                rr = sorted({min(s.R - 1, (tl * 128 + k) // S) for k in (0, 127)})
                probes.update(unit * s.R + r for r in rr)
    for unit in (0, n_units // 2, n_units - 1):
        probes.update(unit * s.R + r for r in range(s.R))
    probes = sorted(i for i in probes if i < c.n)
    assert c.n - 1 in probes and 0 in probes
    dense = out_grads(E, c, seed=61)
    worst = [0.0, 0.0]
    for i in probes:
        gouts = []
        for g in dense:
            zt = torch.zeros_like(g)
            zt[i] = g[i] * c.n
            gouts.append(zt)
        t = backward_state(E, c, s, gouts)
        others = torch.ones(c.n, dtype=torch.bool, device=E.dev)
        others[i] = False
        for name in RAY_INPUTS:
            assert float(t.ing[name][others].abs().max()) == 0.0, (prec, i, name, "gradient on another ray")
        ref, _ = ray_reference(E, c, s, gouts, i)
        pairs = [(k, t.ing[k][i:i + 1] if k in RAY_INPUTS else t.ing[k], ref[k]) for k in ref]
        em, el = check(f"probe ray {i} {prec}", pairs, PROBE_TOL[prec], quiet=True)
        worst = [max(worst[0], em), max(worst[1], el)]
    print(f"{nc}c{nf}f {prec}: {len(probes)} probe rays, others exactly 0; worst max {worst[0]:.2e}, L2 {worst[1]:.2e}")


# ---------------------------------------------------------------------------------------------------------------- edges
def full_backward(E, c, gouts):
    pc, pf = params_of(c)
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=True, inputs=list(RAY_INPUTS) + ["expression"])
    torch.cuda.synchronize()
    return (gc, gf, gl), ing


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("grads", ["mse", "fixed"])
@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("field", ["origin", "direction", "dir_z", "background", "sigma_noise", "out_grad"])
def test_nonfinite_inputs(E, field, bad, grads, prec):
    """A NaN or +inf in one ray's origin, direction, dir_z, background or sigma-noise draw, or in its output gradient, with
    the MSE gradient of nfb_loss_mse_grad or with fixed output gradients that do not depend on the outputs.  Every input and
    parameter gradient float64 autograd makes non-finite is non-finite in the kernel; every other ray's input gradients are
    finite and equal to the clean run's.  (With fixed output gradients a NaN sigma input must still poison its ray: torch's
    ReLU, its compositing and the disparity's max keep NaN.)"""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=70, dir_z=True)
    ray = c.n // 2 + 1
    v = float(bad)
    d = types.SimpleNamespace(**vars(c))
    if field in ("origin", "direction"):
        key = "ro" if field == "origin" else "rd"
        setattr(d, key, getattr(c, key).clone())
        getattr(d, key)[ray, 1] = v
    elif field == "dir_z":
        d.dz = c.dz.clone()
        d.dz[ray] = v
    elif field == "background":
        d.bg = c.bg.clone()
        d.bg[ray, 2] = v
    elif field == "sigma_noise":
        d.noise = dict(c.noise)
        d.noise["n_c"] = c.noise["n_c"].clone()
        d.noise["n_c"][ray, c.nc // 2] = v
    target = torch.rand(c.n, 3, generator=torch.Generator().manual_seed(72)).to(E.dev)

    def run(cc, inject):
        out = train_forward(E, cc)
        s = saved_state(E, cc)
        if grads == "mse":
            gc, gf = torch.zeros(c.n, 3, device=E.dev), torch.zeros(c.n, 3, device=E.dev)
            E.eng.loss_mse_grad(out["rgb_coarse"], out["rgb_fine"], target, c.n, gc, gf, torch.zeros(2, device=E.dev))
            gouts = [gc, None, None, gf, None, None, None]
        else:
            gouts = out_grads(E, cc, seed=71)
        if inject:
            gouts[0] = gouts[0].clone()
            gouts[0][ray, 1] = v
        return s, gouts, full_backward(E, cc, gouts)

    _, _, (_, clean) = run(c, False)
    s, gouts, (kg, ing) = run(d, field == "out_grad")
    ref, R = ray_reference(E, d, s, gouts, ray)
    reached, share = 0, 1.0
    for name, g, r in [(k, ing[k][ray:ray + 1] if k in RAY_INPUTS else ing[k], ref[k]) for k in ref]:
        nonfin = ~torch.isfinite(r)
        reached += int(nonfin.sum())
        assert bool((~torch.isfinite(g[nonfin])).all()), (field, bad, grads, name, "finite where torch gives a non-finite gradient")
    # Parameter gradients: a NaN reaches dW[n, :] through every unit n the ReLU keeps at the bad ray's rows.  Units whose
    # pre-activation is within rounding of 0 there are kept by float64 and dropped by the kernel's FP16 / FP32 records (or the
    # reverse), so entry-wise agreement is not decided; every tensor float64 makes non-finite must be non-finite in the kernel
    # in at least NONFIN_SHARE of those entries (a backward that turns the NaN into a number gives 0).
    for name, g, r in grad_pairs(kg, R):
        nonfin = ~torch.isfinite(r)
        if bool(nonfin.any()):
            reached += int(nonfin.sum())
            frac = float((~torch.isfinite(g[nonfin])).double().mean())
            share = min(share, frac)
            assert frac >= NONFIN_SHARE, (field, bad, grads, name, "finite where torch gives a non-finite gradient", frac)
    assert reached > 0, (field, bad, grads)
    others = torch.ones(c.n, dtype=torch.bool, device=E.dev)
    others[ray] = False
    for name in RAY_INPUTS:
        g, g0 = ing[name][others], clean[name][others]
        assert bool(torch.isfinite(g).all()), (field, bad, grads, name, "another ray's input gradient is non-finite")
        err = float((g - g0).abs().max()) / float(g0.abs().max())
        assert err <= 2e-5, (field, bad, grads, name, err)  # the bad ray may move the power-of-two loss scale
    print(f"{field} = {bad}, {grads} output gradients ({prec}): {reached} entries non-finite in float64; input gradients "
          f"all non-finite in the kernel, parameter gradients at least {share:.4f}; other rays finite")


@pytest.mark.parametrize("prec", PRECS)
def test_chain_fp16_range(E, prec):
    """Weights re-balanced so that the forward and the input gradients are unchanged in exact arithmetic but dY0 and dY3
    reach 0.5x and then 4x FP16's 65504 after the loss scale (layers_xyz.0 and .3 divided by g, the weights of the next
    layers multiplied by g; g from the float64 taps): the input gradients are within IN_TOL of float64 or non-finite,
    never finite and wrong."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=80, dir_z=True)
    gouts = out_grads(E, c, seed=81)
    train_forward(E, c)
    s = saved_state(E, c)
    t = backward_state(E, c, debug_state(E, c), gouts)
    scale = 1.0 / t.inv
    tap = {L: max(float(x.abs().max()) for x in reference(E, c, s.z_c, s.z_f, gouts, want_taps=f"a{L}").taps) for L in (0, 3)}
    base = (c.mc, c.mf)
    for target in (0.5, 4.0):
        gain = {L: target * 65504.0 / (tap[L] * scale) for L in (0, 3)}

        def rebalance(m):
            p = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
            for L in (0, 3):
                p[f"layers_xyz.{L}.weight"] /= gain[L]
                p[f"layers_xyz.{L}.bias"] /= gain[L]
                p[f"layers_xyz.{L + 1}.weight"] *= gain[L]
            return model(E, 0, True, params=p)
        c.mc, c.mf = rebalance(base[0]), rebalance(base[1])
        train_forward(E, c)
        s = debug_state(E, c)
        t = backward_state(E, c, s, gouts)
        recs = dev_tensor(t.dbg.records, (s.n_tiles, t.dbg.record_bytes // 2), "<i2")
        big = {}
        for L in (0, 3):
            img = torch.cat([decode_image(recs, dy_off(L), 256)[rowmap(c, s, pas)] for pas in (0, 1)])
            big[L] = float(img.abs().max()) if bool(torch.isfinite(img).all()) else float("inf")
        ref, _ = reference_inputs(E, c, s.z_c, s.z_f, gouts)
        verdict = []
        for k in ref:
            if not bool(torch.isfinite(t.ing[k]).all()):
                verdict.append(f"{k} non-finite")
                continue
            em, el = check(f"dY x{target} {prec} {k}", [(k, t.ing[k], ref[k])], IN_TOL[prec], quiet=True)
            verdict.append(f"{k} {em:.1e}")
        print(f"{prec}: max |dY0|, |dY3| (scaled) {big[0]:.3g}, {big[3]:.3g} -> {', '.join(verdict)}")
        if target > 1.0:
            assert big[0] == float("inf") and big[3] == float("inf"), big


@pytest.mark.parametrize("prec", PRECS)
def test_loss_scale_is_exact(E, prec):
    """Output gradients times 2^k (k = +-20, +-60) give input, latent and parameter gradients that are bitwise 2^k times the
    unscaled ones: the loss scale is a power of two, the compositing backward is linear in the output gradients, and every
    sum runs in a fixed order, so the FP16 operands of the chain are the same bits."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=82, dir_z=True)
    train_forward(E, c)
    base = out_grads(E, c, seed=83)
    kg0, ing0 = full_backward(E, c, base)
    flat0 = [t for t in list(kg0[0]) + list(kg0[1]) + [kg0[2]] if t is not None] + [ing0[k] for k in sorted(ing0)]
    for k in (-60, -20, 20, 60):
        kg, ing = full_backward(E, c, [g * 2.0 ** k for g in base])
        flat = [t for t in list(kg[0]) + list(kg[1]) + [kg[2]] if t is not None] + [ing[n] for n in sorted(ing)]
        worst = max(float(((a.double() * 2.0 ** k - b.double()).abs() / b.double().abs().max()).max()) for a, b in zip(flat0, flat))
        print(f"{prec}: output gradients x 2^{k}: worst relative difference {worst:.1e}")
        for i, (a, b) in enumerate(zip(flat0, flat)):
            assert torch.equal(a * 2.0 ** k, b), (prec, k, i, worst)


@pytest.mark.parametrize("prec", PRECS)
def test_chunked_against_float64(E, prec, monkeypatch):
    """Over the memory budget (48 MiB: 32 rays per chunk, the last chunk ragged) every input gradient and d latent against
    float64 at the depths of a one-launch forward of the same rays and noise."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=19, dir_z=True)
    train_forward(E, c)
    s = saved_state(E, c)
    gouts = out_grads(E, c, seed=20)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    train_forward(E, c)
    with pytest.raises(RuntimeError, match="train_debug"):  # NFB_ERR_STATE: the buffers only ever hold one chunk
        E.eng.train_debug()
    pc, pf = params_of(c)
    _, _, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=wanted(c))
    torch.cuda.synchronize()
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    ref, R = reference_inputs(E, c, s.z_c, s.z_f, gouts)
    em, el = check(f"chunked {prec} inputs", input_pairs(ing, ref), IN_TOL[prec])
    check(f"chunked {prec} latent", [("latent", gl, R.glat)], TOL[prec])
