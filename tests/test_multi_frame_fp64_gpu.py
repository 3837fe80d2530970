"""The multi-frame path (NFB_MULTI_FRAME: frames_fold_kernel, the per-ray frame lookup of render_frames_kernel, raysum_kernel,
framesum_kernel and frames_grad_kernel of nfb_train.cu §4b, the chunked re-run) against float64, stage by stage, each stage fed
the kernel's own output of the stage before it, read through NfbTrainDebug (frame, frame_table, frame_cond, ray_sums,
frame_sums, records, scale):
  (a) fold           frame_cond[f] bitwise [expression_f / 3 ; latent_f] (FP32 division); every frame_table[net][f] row
                     against float64 bias + W[:, 63:171] c_f from the kernel's own c_f, relative to |bias| + |W| |c_f|; the
                     row after the last frame all NaN.
  (b) frame slots    bitwise the caller's index, n_frames where it was out of range.
  (c) ray sums       ray_sums[pass][g] bitwise the sequential FP32 sum over the ray's samples (ascending) of the decoded dY0 | dY3
                     records times scale[1], and against the float64 sum relative to the sum of absolute values; also against
                     float64 autograd dL/db0, dL/db3 per ray (relative L2 per pass, RAY_L2).
  (d) frame sums     frame_sums[f][pass] bitwise the sequential FP32 sum of the kernel's ray_sums over frame f's rays in
                     ascending order, and against the float64 sum relative to the sum of absolute values.  A frame without
                     rays is exactly 0.
  (e) conditioning   d latent_f and d expression_f against float64 sum_net W0c^T fsum0 + W3c^T fsum3 (expression / 3), and the
                     conditioning columns W0[:, 63:171], W3[:, 63:171] of the parameter gradients against float64
                     sum_f fsum_f (x) frame_cond_f, from the kernel's own frame_sums and frame_cond.
  (f) end to end     against float64 autograd with every ray conditioned on its own frame (torch_reference with
                     per_ray_cond), at the bounds of test_multi_frame_gpu.py; that batched reference equals
                     test_multi_frame_gpu.reference_frames (per frame on the frame's rays).
The stage bounds of (a), (c), (d) and (e) are the worst-case bounds of a k-term FP32 sum, gamma(k) = k u / (1 - k u) with
u = 2^-24, times the sum of absolute values: k = 109 for a folded row, S for a ray of S samples, the frame's ray count for a
frame sum, 256 x networks + 1 for a conditioning gradient (+ 2u for the FP32 1/3), F for a conditioning column.  Every input of
those stages is the kernel's own, so nothing but the order of the FP32 sums may move them.

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases, both precisions and both modes:
  (a) 0.035 of the bound; (c) 0.33 (3c+7f; 0.08 elsewhere); (d) 1.0 with two-ray frames (a single rounding can reach
  u |sum|), 0.06 with more rays; (e) latent / expression 0.008, columns 1.0 at F = 1 (a single rounding), up to 0.89 with 3 to 1024 frames.  The
  bitwise checks of (c) and (d) held in every case.
  (c) ray sums against float64 autograd, relative L2: exact 3.5e-3, fast 4.8e-2          -> RAY_L2 exact 1e-2, fast 1.5e-1
  (f) per-ray input gradients: exact max 6.0e-2, L2 9.1e-3 (white_nobg); fast max 0.16, L2 5.2e-2 -> E2E_IN_TOL.  These exceed
      IN_TOL, which was measured at one conditioning vector: the rays of a frame get the input gradients of the single-frame call
      of that frame (up to the loss scale), and the single-frame nfb_render_backward_ex of white_nobg's frame 0 alone measured
      max 7.1e-2, L2 1.5e-2 on the same rays.  Parameters, latents and expressions stay within TOL / IN_TOL.
  large frames (65,536 rays, chunked under the default budget): per-frame latent / expression against the single-frame
      backward of each frame's rays alone, max / max|ref| 8.5e-5, L2 8.8e-5 as one frame, 4.5e-5, 4.2e-5 as four frames of
      16,384, both precisions: the order of the FP32 sums over 65,536 rays                  -> LARGE_TOL (5e-4, 5e-4)
  chunked, 20-ray frames over 32-ray chunks: end to end exact max 4.7e-3, fast 3.8e-2; drop-in latent table exact 4.2e-4,
      fast 4.0e-3.
The file takes about 45 s on one H100.
Planted defects, each built once (the stage subset: 64c64f, 64c0f, nobg, white_nobg, F217, n513, n1025, prod2048):
  raysum_kernel summing S - 1 samples: (c) bitwise, ~149,000 entries, in the cases without a background image only: with one,
      the last sample's colour is the background and its alpha is 1, so its dY rows are exactly 0 and the defect changes
      nothing.  test_multi_frame_gpu.py: 1 of 28 fails (the drop-in fit, which has no background).
  framesum_kernel skipping position 511 of each 512-ray batch: (d) bitwise, 466-930 entries, every case of 512 rays or more.
      test_multi_frame_gpu.py: 6 of 28 fail (exact mode, the chunked cases and the drop-in, at up to 3.3 times their bounds).
  frames_grad_kernel dropping the fine network's W3c^T fsum3 term: (e) at 3,700-6,800 times the bound; 64c0f passes, having no
      fine network.  test_multi_frame_gpu.py: 9 of 28 fail.
  frames_grad_kernel's conditioning columns taking frame 0's vector for the last frame, or for every frame: (e) at 1e4-2.5e8
      times the bound.  test_multi_frame_gpu.py: 6 of 28 fail for either.
"""
import types

import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_fp64_gpu import E, FAR, NEAR, PROBE_TOL, TOL, TOL_3C_FAST, check, errors, make_case, out_grads  # noqa: F401
from test_backward_fp64_gpu import rowmap, saved_state, two_iter_rays
from test_backward_gpu import decode_image, dev_tensor, dy_off
from test_input_grads_fp64_gpu import bounded, same_bits
from test_input_grads_gpu import IN_TOL, kernel_names, params_of
from test_multi_frame_gpu import EMPTY, frames, param_pairs, reference_frames, render, split_case

pytestmark = pytest.mark.gpu

PRECS = ["exact", "fast"]
ROWS = 512                                  # nfb_layout.h kFrameRows: dY0 (256) | dY3 (256)
RAY_L2 = {"exact": 1e-2, "fast": 1.5e-1}      # per-ray bias sums against float64 autograd, relative L2 per pass
LARGE_TOL = (5e-4, 5e-4)                    # per-frame conditioning, chunked 65,536 rays against single-frame backwards
E2E_IN_TOL = {"exact": (1e-1, 2e-2), "fast": (3e-1, 1e-1)}  # per-ray input gradients end to end (module docstring)
U = 2.0 ** -24


def gamma(k):
    return k * U / (1.0 - k * U)


def wanted(c):
    return ["ray_origins", "ray_directions", "expression"] + (["background"] if c.bg is not None else []) + \
        (["dir_z"] if c.dz is not None else [])


def layout(kind, n, nfr, seed=0):
    """Frame index [n] (CPU int32): a random interleave leaving frame EMPTY without rays (when nfr > EMPTY), contiguous blocks
    as a data loader yields them, rays on the first and last frame only, every ray its own frame, or 512-ray batches (frame b
    holds the rays of batch b of framesum_kernel)."""
    g = torch.Generator().manual_seed(300 + seed)
    if kind == "interleave":
        used = torch.tensor([f for f in range(nfr) if nfr <= EMPTY or f != EMPTY])
        fi = used[torch.randint(0, len(used), (n,), generator=g)]
    elif kind == "blocks":
        fi = torch.arange(n) * nfr // n
    elif kind == "ends":
        fi = torch.where(torch.rand(n, generator=g) < 0.5, 0, nfr - 1)
    elif kind == "own":
        assert nfr == n
        fi = torch.arange(n)
    elif kind == "batches":
        fi = torch.arange(n) // 512
        assert int(fi.max()) < nfr
    else:
        raise ValueError(kind)
    return fi.to(torch.int32)


# ---------------------------------------------------------------------------------------------------------------- state
def frame_state(E, c):
    """NfbTrainDebug's multi-frame fields after a one-launch multi-frame training forward (sums: None until a backward)."""
    torch.cuda.synchronize()
    d = E.eng.train_debug()
    F, npass = d.n_frames, 2 if c.nf else 1
    st = types.SimpleNamespace(F=F, dbg=d)
    st.frame = dev_tensor(d.frame, (c.n,), "<i4").clone()
    st.tab = [dev_tensor(d.frame_table[k], (F + 1, ROWS)).clone() for k in range(npass)]
    assert (d.frame_table[1] is None) == (npass == 1)
    st.cond = dev_tensor(d.frame_cond, (F, 108)).clone()
    return st


def sums_state(E, c, st):
    torch.cuda.synchronize()
    d = E.eng.train_debug()
    assert d.ray_sums and d.frame_sums
    npass = 2 if c.nf else 1
    t = types.SimpleNamespace(dbg=d, inv=float(dev_tensor(d.scale, (2,))[1]))
    t.raysum = dev_tensor(d.ray_sums, (npass, c.n, ROWS)).clone()
    t.fsum = dev_tensor(d.frame_sums, (st.F, 2, ROWS)).clone()
    return t


def models(c):
    return [c.mc] + ([c.mf] if c.nf else [])


def cond_weights(m):
    P = dict(m.named_parameters())
    return [(P[f"layers_xyz.{L}.weight"].detach().double()[:, 63:171], P[f"layers_xyz.{L}.bias"].detach().double()) for L in (0, 3)]


# ---------------------------------------------------------------------------------------------------------------- (a), (b)
def check_fold(c, ex, la, st, tag):
    want = torch.cat(((ex.double() / 3.0).float(), la.float()), 1)  # a division of FP32 values, rounded once
    assert same_bits(st.cond, want), (tag, "frame_cond")
    cd = st.cond.double()
    worst = 0.0
    for net, m in enumerate(models(c)):
        (W0, b0), (W3, b3) = cond_weights(m)
        ref = torch.cat((b0 + cd @ W0.t(), b3 + cd @ W3.t()), 1)
        mag = torch.cat((b0.abs() + cd.abs() @ W0.abs().t(), b3.abs() + cd.abs() @ W3.abs().t()), 1)
        w, _ = bounded(f"{tag} frame_table[{net}]", st.tab[net][:st.F], ref, mag * gamma(109), 1.0)
        worst = max(worst, w)
        assert bool(torch.isnan(st.tab[net][st.F]).all()), (tag, net, "the row after the last frame")
    return worst


def check_slots(fi, st, tag):
    want = fi.long().clone()
    want[(want < 0) | (want >= st.F)] = st.F
    assert torch.equal(st.frame.long().cpu(), want), tag


# ---------------------------------------------------------------------------------------------------------------- (c)
def dy_rows(E, c, s, t):
    """Per pass [n, S, 512]: the decoded FP16 dY0 | dY3 records of every (ray, sample) row, loss-scaled."""
    recs = dev_tensor(t.dbg.records, (s.n_tiles, t.dbg.record_bytes // 2), "<i2")
    imgs = [decode_image(recs, dy_off(L), 256) for L in (0, 3)]
    out = []
    for pas in range(2 if c.nf else 1):
        tile, row = rowmap(c, s, pas)
        S = c.nc + c.nf if pas else c.nc
        out.append(torch.cat([img[tile, row] for img in imgs], 1).view(c.n, S, ROWS))
    return out


def check_raysums(E, c, s, t, tag, valid, db64=None, dy=None):
    """dy: per pass the dY0 | dY3 rows raysum read, [n, S, 512] (by default the FP16 records; exact-grad passes hi + lo)."""
    worst, l2 = 0.0, 0.0
    for pas, x in enumerate(dy_rows(E, c, s, t) if dy is None else dy):
        got = t.raysum[pas]
        acc = torch.zeros(c.n, ROWS, device=x.device)
        for i in range(x.shape[1]):  # raysum_kernel's order: samples ascending, FP32, then the inverse scale (a power of two)
            acc = acc + x[:, i]
        emu = acc * t.inv
        assert torch.equal(got[valid], emu[valid]), (tag, pas, "ray_sums differ from the sequential FP32 sum",
                                                     int((got[valid] != emu[valid]).sum()))
        xd = x[valid].double()
        w, _ = bounded(f"{tag} ray_sums pass {pas}", got[valid], xd.sum(1) * t.inv, xd.abs().sum(1) * t.inv * gamma(x.shape[1]), 1.0)
        worst = max(worst, w)
        if db64 is not None:
            em, el = errors(got[valid], db64[pas][valid])
            l2 = max(l2, el)
            assert el <= (RAY_L2[c.prec] if valid.sum() > 3 else PROBE_TOL[c.prec][1]), (tag, pas, "ray_sums vs dL/db", em, el)
    return worst, l2


# ---------------------------------------------------------------------------------------------------------------- (d)
def check_framesums(c, st, t, tag):
    F, n = st.F, c.n
    slot = st.frame.long()
    valid = slot < F
    rays = torch.arange(n, device=slot.device)[valid]
    fr = slot[valid]
    counts = torch.bincount(fr, minlength=F)
    # the rays of each frame in ascending order, padded with an index of an all-zero row
    order = torch.argsort(fr * n + rays)
    fr_s, rays_s = fr[order], rays[order]
    start = torch.cumsum(counts, 0) - counts
    rank = torch.arange(len(fr_s), device=slot.device) - start[fr_s]
    M = int(counts.max()) if len(fr_s) else 0
    idx = torch.full((F, max(M, 1)), n, dtype=torch.long, device=slot.device)
    idx[fr_s, rank] = rays_s
    worst = 0.0
    for pas in range(2 if c.nf else 1):
        rs = torch.cat((t.raysum[pas], torch.zeros(1, ROWS, device=slot.device)))
        acc = torch.zeros(F, ROWS, device=slot.device)
        for k in range(M):
            acc = acc + rs[idx[:, k]]
        got = t.fsum[:, pas]
        assert torch.equal(got, acc), (tag, pas, "frame_sums differ from the sequential FP32 sum over the frame's rays",
                                       int((got != acc).sum()))
        ref = torch.zeros(F, ROWS, dtype=torch.float64, device=slot.device).index_add_(0, fr, t.raysum[pas][valid].double())
        mag = torch.zeros_like(ref).index_add_(0, fr, t.raysum[pas][valid].double().abs())
        k = (counts - 1).clamp(min=1).double().view(F, 1)
        w, _ = bounded(f"{tag} frame_sums pass {pas}", got, ref, mag * k * U / (1.0 - k * U), 1.0)
        worst = max(worst, w)
        assert int(torch.count_nonzero(got[counts == 0])) == 0, (tag, pas, "a frame without rays")
    return worst


# ---------------------------------------------------------------------------------------------------------------- (e)
def check_cond_grads(c, st, t, glat, gexp, tag):
    fs = t.fsum.double()
    v = torch.zeros(st.F, 108, dtype=torch.float64, device=fs.device)
    a = torch.zeros_like(v)
    nets = models(c)
    for net, m in enumerate(nets):
        (W0, _), (W3, _) = cond_weights(m)
        b0, b3 = fs[:, net, :256], fs[:, net, 256:]
        v += b0 @ W0 + b3 @ W3
        a += b0.abs() @ W0.abs() + b3.abs() @ W3.abs()
    g = gamma(256 * len(nets) + 1)
    worst = 0.0
    if gexp is not None:
        worst = max(worst, bounded(f"{tag} d expression", gexp, v[:, :76] / 3.0, a[:, :76] / 3.0 * (g + 2 * U), 1.0)[0])
    if glat is not None:
        worst = max(worst, bounded(f"{tag} d latent", glat, v[:, 76:], a[:, 76:] * g, 1.0)[0])
    return worst


def check_cond_columns(c, st, t, gc, gf, tag):
    fs, cd = t.fsum.double(), st.cond.double()
    worst = 0.0
    for net, gs in enumerate([gc] + ([gf] if c.nf else [])):
        for L, i in ((0, 0), (1, 6)):
            b = fs[:, net, 256 * L:256 * L + 256]
            got = gs[i][:, 63:171]
            worst = max(worst, bounded(f"{tag} conditioning columns {net}/{i}", got, b.t() @ cd, b.abs().t() @ cd.abs() * gamma(st.F),
                                       1.0)[0])
    return worst


# ---------------------------------------------------------------------------------------------------------------- float64
def reference_multi(E, c, fi, ex, la, z_c, z_f, gouts, sel=None):
    """float64 autograd of sum_i <out_i, gouts_i> over the rays `sel` (all by default), each ray conditioned on its own frame
    through ex[fi], la[fi]: parameter gradients, d latent [F,32], d expression [F,76], input gradients per ray (0 outside sel), and
    per pass the per-ray bias gradients [n, 512] = (dL/db0 | dL/db3) of that ray's samples."""
    dev = E.dev
    f64 = lambda t: None if t is None else t.detach().to(dev, torch.float64)  # noqa: E731
    leaf = lambda t: None if t is None else f64(t).requires_grad_(True)  # noqa: E731
    pc = {k: leaf(v) for k, v in c.mc.named_parameters()}
    pf = {k: leaf(v) for k, v in c.mf.named_parameters()} if c.nf else None
    ro, rd, bg, dz, ex64, la64 = leaf(c.ro), leaf(c.rd), leaf(c.bg), leaf(c.dz), leaf(ex), leaf(la)
    fi = fi.to(dev).long()
    sel = torch.arange(c.n, device=dev) if sel is None else sel.to(dev)
    npass = 2 if c.nf else 1
    db = torch.zeros(npass, c.n, ROWS, dtype=torch.float64, device=dev)
    nearfar = torch.tensor([NEAR, FAR], device=dev, dtype=torch.float64).expand(c.n, 2)
    chunk = max(16, 32768 // (2 * c.nc + c.nf))
    for b in range(0, len(sel), chunk):
        r = sel[b:b + chunk]
        taps = {}
        o = TR.render_at_depths(torch.cat((ro[r], rd[r], nearfar[r]), -1), pc, pf, ex64[fi[r]], la64[fi[r]], f64(z_c[r]),
                                f64(z_f[r]) if c.nf else None, NEAR, FAR, c.noise_std, {k: f64(v[r]) for k, v in c.noise.items()},
                                c.white, bg[r] if bg is not None else None, dz[r] if dz is not None else None, taps, per_ray_cond=True)
        loss = sum(((oi * f64(gi[r])).sum() for oi, gi in zip(o, gouts) if oi is not None and gi is not None),
                   torch.zeros((), dtype=torch.float64, device=dev))
        loss.backward()
        for pas, key in enumerate(("coarse", "fine")[:npass]):
            S = c.nc + c.nf if pas else c.nc
            for L in (0, 3):
                db[pas, r, 256 * (L // 3):256 * (L // 3) + 256] = taps[key][f"a{L}"].grad.view(len(r), S, 256).sum(1)
    z = lambda t, like: t.grad if t.grad is not None else torch.zeros_like(like)  # noqa: E731
    ins = dict(ray_origins=z(ro, ro), ray_directions=z(rd, rd))
    if bg is not None:
        ins["background"] = z(bg, bg)
    if dz is not None:
        ins["dir_z"] = z(dz, dz)
    return types.SimpleNamespace(gc=[pc[k].grad for k in TR.PARAM_ORDER], gf=[pf[k].grad for k in TR.PARAM_ORDER] if pf else None,
                                 glat=z(la64, la64), gexp=z(ex64, ex64), ins=ins, db=db)


def e2e_tols(c, fi):
    """(latent, expression, per-ray input) bounds: those of test_multi_frame_gpu.py, single-ray bounds with 1-3 rays, the input
    bounds for the latent table when the frames hold fewer than 16 rays each on average (few-ray gradients, like per-ray input
    gradients), and E2E_IN_TOL for the per-ray input gradients."""
    if c.n <= 3:
        return PROBE_TOL[c.prec], PROBE_TOL[c.prec], PROBE_TOL[c.prec]
    tol = TOL_3C_FAST if (c.nc, c.prec) == (3, "fast") else TOL[c.prec]
    used = int(torch.unique(fi).numel())
    return (tol if c.n >= 16 * used else IN_TOL[c.prec]), IN_TOL[c.prec], E2E_IN_TOL[c.prec]


def check_end_to_end(c, fi, kg, ing, R, tag, want_params, rays=None):
    tol, ex_tol, in_tol = e2e_tols(c, fi)
    gc, gf, gl = kg
    worst = [0.0, 0.0]
    pick = (lambda t: t) if rays is None else (lambda t: t[rays])  # noqa: E731
    if want_params:
        worst = check(f"{tag} params", param_pairs(gc, gf, R.gc, R.gf), TOL_3C_FAST if (c.nc, c.prec) == (3, "fast") else
                      (TOL[c.prec] if c.n > 3 else PROBE_TOL[c.prec]), quiet=True)
    for name, got, ref, tl in [("latent", gl, R.glat, tol), ("expression", ing["expression"], R.gexp, ex_tol)] + \
            [(k, pick(ing[k]), pick(R.ins[k]), in_tol) for k in R.ins]:
        em, el = check(f"{tag} {name}", [(name, got, ref)], tl, quiet=True)
        worst = [max(worst[0], em), max(worst[1], el)]
    return worst


# ---------------------------------------------------------------------------------------------------------------- cases
def run_stages(E, c, nfr, kind, tag, seed=0, cross_check=False):
    ex, la = frames(E, nfr, seed)
    fi = layout(kind, c.n, nfr, seed)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    s = saved_state(E, c)
    st = frame_state(E, c)
    assert st.F == nfr
    check_slots(fi, st, tag)
    fold = check_fold(c, ex, la, st, tag)
    gouts = out_grads(E, c)
    R = reference_multi(E, c, fi, ex, la, s.z_c, s.z_f, gouts)
    if cross_check:  # the batched float64 reference is test_multi_frame_gpu's per-frame one
        rc, rf, rlat, rexp, rins = reference_frames(E, c, fi, nfr, ex, la, s.z_c, s.z_f, gouts)
        for a, b in [(R.glat, rlat), (R.gexp, rexp)] + [(R.ins[k], rins[k]) for k in rins] + \
                [(x, y) for x, y in zip(R.gc + (R.gf or []), rc + (rf or [])) if x is not None]:
            assert float((a - b).abs().max()) <= 1e-9 * float(b.abs().max()) + 1e-300, tag
    valid = torch.ones(c.n, dtype=torch.bool, device=E.dev)
    pc, pf = params_of(c)
    res = {}
    for mode in ("input_only", "full"):
        gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=mode == "full", inputs=wanted(c), frames=True)
        t = sums_state(E, c, st)
        rsum, rl2 = check_raysums(E, c, s, t, f"{tag} {mode}", valid, R.db)
        fsum = check_framesums(c, st, t, f"{tag} {mode}")
        cond = check_cond_grads(c, st, t, gl, ing["expression"], f"{tag} {mode}")
        cols = check_cond_columns(c, st, t, gc, gf, f"{tag} {mode}") if mode == "full" else 0.0
        e2e = check_end_to_end(c, fi, (gc, gf, gl), ing, R, f"{tag} {mode}", mode == "full")
        res[mode] = (t, gl, ing)
        print(f"{tag} {mode}: share of the gamma bound: fold {fold:.2e}, ray sums {rsum:.2e}, frame sums {fsum:.2e}, latent / "
              f"expression {cond:.2e}, columns {cols:.2e}; ray sums against float64 L2 {rl2:.2e}; end to end max {e2e[0]:.1e} "
              f"L2 {e2e[1]:.1e}")
    (t0, l0, i0), (t1, l1, i1) = res["input_only"], res["full"]
    assert torch.equal(t0.raysum, t1.raysum) and torch.equal(t0.fsum, t1.fsum) and torch.equal(l0, l1), tag
    assert all(torch.equal(i0[k], i1[k]) for k in i0), tag


def _case(nc=64, nf=64, n=None, nfr=5, kind="interleave", stress=True, seed=0, cross=False, **kw):
    def make(E, prec):
        return make_case(E, two_iter_rays(E) if n is None else n, nc, nf, prec, stress=stress, seed=seed, **kw), nfr, kind, cross
    return make


CASES = {
    # sample geometries (4 * SMs + 37 rays: every CTA runs two units, the last unit half filled), 5 frames, frame 3 empty
    "64c64f": _case(dir_z=True, seed=1, cross=True),
    "64c128f": _case(64, 128, seed=2),
    "128c256f": _case(128, 256, seed=3),
    "3c7f": _case(3, 7, seed=4),
    "64c0f": _case(64, 0, seed=5, cross=True),
    # compositing options
    "nobg": _case(bg=False, seed=6),
    "white_nobg": _case(bg=False, white=True, seed=7),
    "noise_off": _case(perturb=False, noise_std=0.0, seed=8),
    # frame counts (frames_grad_kernel: 216 column blocks, then one block per frame) and layouts
    "F1_all_rays": _case(nfr=1, seed=9),
    "F216_blocks": _case(nfr=216, kind="blocks", seed=10),
    "F217_blocks": _case(nfr=217, kind="blocks", seed=11),
    "F1024_ends": _case(nfr=1024, kind="ends", seed=12),
    "F1024x2_2048": _case(n=2048, nfr=1024, kind="blocks", stress=False, seed=13),
    "prod2048_F8": _case(n=2048, nfr=8, stress=False, seed=14),
    # ray counts at framesum_kernel's 512-ray batches
    "n1": _case(n=1, seed=15),
    "n511": _case(n=511, seed=16),
    "n512": _case(n=512, seed=17),
    "n513_own_frames": _case(n=513, nfr=513, kind="own", seed=18),   # one-ray frames; frame 512 in the partial last batch
    "n1025_batches": _case(n=1025, nfr=3, kind="batches", seed=19),  # two full 512-ray lists, then one ray at position 1024
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(CASES))
def test_multi_frame_stages_against_float64(E, case, prec):
    c, nfr, kind, cross = CASES[case](E, prec)
    run_stages(E, c, nfr, kind, f"{case} {prec}", cross_check=cross)


# ---------------------------------------------------------------------------------------------------------------- hook
def test_debug_hook_fields(E):
    """After a single-frame training forward: n_frames 0 and NULL frame pointers.  After a multi-frame one: the tables, and
    the sums NULL until a backward formed them (an input-only backward too, with no weight-gradient launch); a chunked forward
    is NFB_ERR_STATE."""
    c = make_case(E, 300, 64, 64, "fast", seed=30)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    render(E, c, True)
    d = E.eng.train_debug()
    assert d.n_frames == 0 and not d.frame and not d.frame_table[0] and not d.frame_table[1] and not d.frame_cond
    assert not d.ray_sums and not d.frame_sums
    ex, la = frames(E, 4)
    E.eng.set_frames(ex, la)
    fi = layout("interleave", c.n, 4)
    render(E, c, True, fi)
    d = E.eng.train_debug()
    assert d.n_frames == 4 and d.frame and d.frame_table[0] and d.frame_table[1] and d.frame_cond
    assert not d.ray_sums and not d.frame_sums
    pc, pf = params_of(c)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        E.eng.backward(list(out_grads(E, c)), pc, pf, want_params=False, inputs=["expression"], frames=True)
        torch.cuda.synchronize()
    names = kernel_names(prof)
    assert any("raysum_kernel" in k for k in names) and any("framesum_kernel" in k for k in names), names
    assert not any("dw_kernel" in k for k in names), names
    d = E.eng.train_debug()
    assert d.ray_sums and d.frame_sums
    render(E, c, True, fi)
    d = E.eng.train_debug()
    assert not d.ray_sums and not d.frame_sums


# ---------------------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("prec", PRECS)
def test_chunked_frames_straddle_chunks(E, prec, monkeypatch):
    """48 MiB = 32 rays per chunk; contiguous frames of 20 rays straddle chunk boundaries, and the last frame (rays 560..564)
    lies in the ragged last chunk only.  Against float64 (depths of a one-launch forward of the same rays and noise) and per
    ray within 1e-3 of the one-launch backward of that forward."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=40, dir_z=True)
    nfr = (c.n + 19) // 20
    fi = (torch.arange(c.n) // 20).to(torch.int32).to(E.dev)
    assert c.n % 32 != 0 and (nfr - 1) * 20 >= (c.n - 1) // 32 * 32  # the last frame starts inside the last chunk
    ex, la = frames(E, nfr, 4)
    gouts = out_grads(E, c, seed=41)
    pc, pf = params_of(c)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    s = saved_state(E, c)
    one = E.eng.backward(list(gouts), pc, pf, inputs=wanted(c), frames=True)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    with pytest.raises(RuntimeError, match="train_debug"):
        E.eng.train_debug()
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, inputs=wanted(c), frames=True)
    torch.cuda.synchronize()
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    for k in ing:
        em, el = errors(ing[k], one[3][k])
        assert em <= 1e-3 and el <= 1e-3, (k, em, el)
    em, el = errors(gl, one[2])
    assert em <= 1e-3 and el <= 1e-3, ("latent", em, el)
    R = reference_multi(E, c, fi, ex, la, s.z_c, s.z_f, gouts)
    e2e = check_end_to_end(c, fi.cpu(), (gc, gf, gl), ing, R, f"chunked {prec}", True)
    assert int(torch.count_nonzero(gl[nfr - 1])) > 0
    print(f"chunked {prec}: {nfr} frames of 20 rays over 32-ray chunks; end to end max {e2e[0]:.1e}, L2 {e2e[1]:.1e}")


def big_case(E, n, prec, seed):
    """n rays (the 48 x 48 frame's rays repeated, directions jittered), perturbation, sigma noise and a background."""
    c = make_case(E, 1, 64, 64, prec, stress=False, seed=seed)
    g = torch.Generator().manual_seed(2000 + seed)
    k = torch.arange(n) % E.ro.shape[0]
    c.n = n
    c.ro = E.ro[k.to(E.dev)].contiguous()
    c.rd = (E.rd[k.to(E.dev)] + 0.01 * torch.randn(n, 3, generator=g).to(E.dev)).contiguous()
    c.bg = E.bg[k.to(E.dev)].contiguous()
    nz = O.draw_noise(n, O.Sampling(64, 64, True, 0.1, False, 2048), g)
    c.noise = {key: getattr(nz, key).to(E.dev) for key in ("t_rand", "n_c", "u", "n_f") if getattr(nz, key) is not None}
    return c


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("nfr", [1, 4])
def test_large_frames_against_single_frame(E, nfr, prec):
    """65,536 rays as 1 frame or 4 frames of 16,384 (over the default memory budget: the chunked path).  Each frame's latent
    and expression against nfb_render_backward_ex over that frame's rays alone, which sums in another order (the bias totals of
    the weight-gradient reduction, other chunks and loss scales): the sequential FP32 per-frame sum at fitting sizes."""
    n = 65536
    c = big_case(E, n, prec, seed=50 + nfr)
    ex, la = frames(E, nfr, 5)
    fi = (torch.arange(n) // (n // nfr)).to(torch.int32).to(E.dev)
    gouts = out_grads(E, c, seed=51)
    pc, pf = params_of(c)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    with pytest.raises(RuntimeError, match="train_debug"):  # chunked
        E.eng.train_debug()
    _, _, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["expression"], frames=True)
    torch.cuda.synchronize()
    gl, gx = gl.clone(), ing["expression"].clone()
    worst = [0.0, 0.0]
    for f in range(nfr):
        idx = torch.nonzero(fi == f).flatten()
        cf = split_case(c, idx, ex[f], la[f])
        E.eng.set_frame(ex[f], la[f])
        render(E, cf, True)
        _, _, gl1, ing1 = E.eng.backward([g[idx] if g is not None else None for g in gouts], pc, pf, want_params=False,
                                         inputs=["expression"])
        torch.cuda.synchronize()
        for name, got, ref in (("latent", gl[f], gl1), ("expression", gx[f], ing1["expression"])):
            em, el = errors(got, ref)
            worst = [max(worst[0], em), max(worst[1], el)]
    print(f"{n} rays as {nfr} frame(s), {prec}: per-frame latent / expression against single-frame backwards: max {worst[0]:.2e}, "
          f"L2 {worst[1]:.2e}")
    assert worst[0] <= LARGE_TOL[0] and worst[1] <= LARGE_TOL[1], worst


@pytest.mark.parametrize("prec", PRECS)
def test_single_frame_backward_of_multi_frame_forward(E, prec):
    """nfb_render_backward_ex after a multi-frame forward, asked for neither latent nor expression: parameter and input
    gradients bit-identical to nfb_render_backward_frames of the same forward (nfb.h: "the other gradients are formed as here"),
    in full and in input-only mode."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=60, dir_z=True)
    ex, la = frames(E, 5, 6)
    fi = layout("interleave", c.n, 5, 6)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    gouts = out_grads(E, c, seed=61)
    pc, pf = params_of(c)
    inputs = [k for k in wanted(c) if k != "expression"]
    for want_params in (True, False):
        a = E.eng.backward(list(gouts), pc, pf, want_params=want_params, inputs=inputs, frames=True)
        b = E.eng.backward(list(gouts), pc, pf, want_latent=False, want_params=want_params, inputs=inputs)
        torch.cuda.synchronize()
        if want_params:
            for x, y in zip(list(a[0]) + list(a[1]), list(b[0]) + list(b[1])):
                assert (x is None and y is None) or torch.equal(x, y)
        assert b[2] is None and all(torch.equal(a[3][k], b[3][k]) for k in inputs)


@pytest.mark.parametrize("prec", PRECS)
def test_out_of_range_frames_in_training(E, prec):
    """Indices -1, F, INT32_MAX and INT32_MIN on four rays of a training forward: those rays render NaN and save frame slot F.
    The other rays' input gradients are finite and equal float64 on those rays alone; every frame's latent and expression are
    finite and equal float64 over the in-range rays, and its frame sums are the sums over its own rays (the bad rays' NaN reaches
    neither them nor the loss scale); the bad rays' own input gradients are non-finite, and so are the parameter gradients."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=70, dir_z=True)
    nfr = 5
    ex, la = frames(E, nfr, 7)
    fi = layout("interleave", c.n, nfr, 7)
    bad = torch.tensor([3, 100, c.n // 2, c.n - 1])
    fi[bad] = torch.tensor([-1, nfr, 2 ** 31 - 1, -2 ** 31], dtype=torch.int32)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    out = render(E, c, True, fi)
    s = saved_state(E, c)
    st = frame_state(E, c)
    check_slots(fi, st, "out of range")
    good = torch.ones(c.n, dtype=torch.bool)
    good[bad] = False
    assert bool(torch.isnan(out["rgb_fine"][bad.to(E.dev)]).all()) and bool(torch.isfinite(out["rgb_fine"][good.to(E.dev)]).all())
    gouts = out_grads(E, c, seed=71)
    pc, pf = params_of(c)
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, inputs=wanted(c), frames=True)
    t = sums_state(E, c, st)
    gd = good.to(E.dev)
    fi_good = fi.clone()
    fi_good[bad] = 0  # unused: the reference covers the good rays only
    R = reference_multi(E, c, fi_good, ex, la, s.z_c, s.z_f, gouts, sel=torch.nonzero(gd).flatten())
    check_raysums(E, c, s, t, f"out of range {prec}", gd, R.db)
    check_framesums(c, st, t, f"out of range {prec}")
    check_cond_grads(c, st, t, gl, ing["expression"], f"out of range {prec}")
    assert bool(torch.isfinite(gl).all()) and bool(torch.isfinite(ing["expression"]).all())
    for k in ing:
        if k != "expression":
            assert not bool(torch.isfinite(ing[k][~gd]).any()), (k, "a bad ray's input gradient is finite")
            assert bool(torch.isfinite(ing[k][gd]).all()), (k, "a good ray's input gradient is not finite")
    check_end_to_end(c, fi[good], (gc, gf, gl), ing, R, f"out of range {prec}", False, rays=gd)
    for net, gs in (("coarse", gc), ("fine", gf)):
        assert any(not bool(torch.isfinite(g).all()) for g in gs if g is not None), (net, "parameter gradients all finite")


def test_reloaded_weights_make_frames_stale(E):
    """nfb_load_weights (sync_weights with other parameters) or nfb_repack after nfb_set_frames: a multi-frame render is
    NFB_ERR_STATE until nfb_set_frames runs again."""
    c = make_case(E, 64, 64, 64, "fast", seed=80)
    ex, la = frames(E, 3)
    fi = layout("interleave", c.n, 3)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    ref = render(E, c, False, fi)["rgb_fine"].clone()
    other = make_case(E, 64, 64, 64, "fast", stress=False, seed=80)
    E.eng.sync_weights(other.mc, c.mf)
    with pytest.raises(RuntimeError, match="render_forward_frames"):
        render(E, c, False, fi)
    with pytest.raises(RuntimeError, match="render_forward_frames"):
        render(E, c, True, fi)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    assert torch.equal(render(E, c, False, fi)["rgb_fine"], ref)
    pc, pf = params_of(c)
    E.eng.repack([p.detach().contiguous() for p in pc], [p.detach().contiguous() for p in pf])
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="render_forward_frames"):
        render(E, c, False, fi)
    E.eng.set_frames(ex, la)
    assert torch.equal(render(E, c, False, fi)["rgb_fine"], ref)


@pytest.mark.parametrize("prec", PRECS)
def test_dropin_latent_table_chunked(E, prec, monkeypatch):
    """nerf.render_frames under autograd over the memory budget (the chunked path), 6 frames sharing a 3-row latent table
    through latent_table[ids], a temporary int64 frame index: d latent_table and d expressions against float64.  The forward
    keeps its int32 copy of the frame index alive for the chunked backward, whatever the caller frees in between."""
    nerf = E.nerf
    c = make_case(E, two_iter_rays(E), 32, 32, prec, seed=90, perturb=False, noise_std=0.0, bg=False)
    for p in list(c.mc.parameters()) + list(c.mf.parameters()):
        p.requires_grad_(False)
    opts = types.SimpleNamespace(
        dataset=types.SimpleNamespace(no_ndc=True, near=NEAR, far=FAR),
        nerf=types.SimpleNamespace(train=types.SimpleNamespace(num_coarse=32, num_fine=32, perturb=False, lindisp=False,
                                                               radiance_field_noise_std=0.0, white_background=False, chunksize=512)))
    nfr = 6
    ex0, la0 = frames(E, nfr, 8)
    table = la0[:3].clone().requires_grad_(True)
    expr = ex0.clone().requires_grad_(True)
    ids = torch.tensor([0, 1, 2, 2, 1, 0], device=E.dev)
    gouts = out_grads(E, c, seed=91)
    # depths: a one-launch training forward of the same rays (deterministic sampling)
    fi_ref = (torch.arange(c.n) % nfr).to(torch.int32)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex0, table.detach()[ids])
    render(E, c, True, fi_ref)
    s = saved_state(E, c)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    old = nerf.get_precision()
    nerf.set_precision(prec)
    try:
        out = nerf.render_frames(c.ro, c.rd, torch.arange(c.n, device=E.dev) % nfr, expr, table[ids], c.mc, c.mf, opts)
        junk = [torch.full((1 << 20,), -7, dtype=torch.int64, device=E.dev) for _ in range(8)]  # reuse freed blocks
        loss = sum((o * g).sum() for o, g in zip(out, gouts) if o is not None and g is not None)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        nerf.set_precision(old)
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    del junk
    R = reference_multi(E, c, fi_ref, ex0, table.detach()[ids], s.z_c, s.z_f, gouts)
    gtab = torch.zeros(3, 32, dtype=torch.float64, device=E.dev).index_add_(0, ids, R.glat)
    check(f"drop-in chunked {prec}", [("latent_table", table.grad, gtab)], TOL[prec])
    check(f"drop-in chunked {prec}", [("expressions", expr.grad, R.gexp)], IN_TOL[prec])
