"""Several frames in one call (NFB_MULTI_FRAME: nfb_set_frames, nfb_render_forward_frames[_train], nfb_render_backward_frames,
nerf.render_frames).

Forward: every ray of a multi-frame call renders bit for bit as the single-frame call of its own frame renders it (the same
full ray array, the same noise).  Backward: against the float64 restatement (tests/torch_reference.py) evaluated per frame on
that frame's rays, the parameter gradients summed over frames, at the tolerances of test_backward_fp64_gpu.py /
test_input_grads_gpu.py."""
import ctypes as C
import types

import pytest
import torch

import torch_reference as TR
from test_backward_fp64_gpu import E, FAR, NEAR  # noqa: F401
from test_backward_fp64_gpu import PRECS, TOL, check, errors, make_case, out_grads, saved_state, two_iter_rays
from test_backward_fp64_gpu import rowmap
from test_backward_gpu import dev_tensor
from test_input_grads_gpu import IN_TOL, reference_inputs

pytestmark = pytest.mark.gpu

OUTS = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
F = 5
EMPTY = 3  # a frame no ray uses


def frames(E, nfr, seed=0):
    g = torch.Generator().manual_seed(77 + seed)
    ex = (E.expr.cpu().reshape(1, 76) + 0.5 * torch.randn(nfr, 76, generator=g)).to(E.dev)
    la = (E.latent.cpu().reshape(1, 32) + 0.5 * torch.randn(nfr, 32, generator=g)).to(E.dev)
    return ex.contiguous(), la.contiguous()


def frame_index(n, nfr, seed=0, empty=EMPTY):
    """An arbitrary interleaving (so units and tiles mix frames) that leaves frame `empty` without rays."""
    g = torch.Generator().manual_seed(5 + seed)
    used = torch.tensor([f for f in range(nfr) if f != empty])
    return used[torch.randint(0, len(used), (n,), generator=g)].to(torch.int32)


def render(E, c, train, fi=None):
    E.eng.sync_weights(c.mc, c.mf)
    return E.eng.render(c.ro, c.rd, NEAR, FAR, c.nc, c.nf, perturb=c.perturb, noise_std=c.noise_std, white_bkgd=c.white,
                        background=c.bg, dir_z=c.dz, noise=c.noise, precision=c.prec, train=train,
                        frame_index=fi.to(E.dev) if fi is not None else None)


def params_of(c):
    pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
    pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER] if c.mf is not None else None
    return pc, pf


# The per-row content of a training record (nfb_layout.h kRec*): every transposed FP16 image the forward writes (PE, h0..h5,
# g0..g2, direction encoding) as (byte offset, features), and the nine ReLU-mask words of each layer.
REC_IMAGES = [(0, 64)] + [(16384 + 65536 * l, 256) for l in range(6)] + [(16384 + 6 * 65536 + 32768 * l, 128) for l in range(3)] + \
    [(16384 + 6 * 65536 + 3 * 32768, 32)]
REC_MASK = 16384 + 6 * 65536 + 3 * 32768 + 8192


def record_rows(E, c):
    """[rows, features] FP16 bits and [rows, 72] mask words of every (pass, ray, sample) row of the last training forward, rows in
    the order (pass, ray, sample)."""
    s = saved_state(E, c)
    recs = dev_tensor(s.dbg.records, (s.n_tiles * s.dbg.record_bytes,), "|u1")
    h16, masks = [], []
    for pas in range(2 if c.nf else 1):
        tile, r = rowmap(c, s, pas)
        base = tile.long() * s.dbg.record_bytes
        r = r.long().view(-1, 1)
        cols = []
        for off, nfeat in REC_IMAGES:
            k = torch.arange(nfeat, device=E.dev).view(1, -1)
            r63 = r & 63
            o = (r >> 6) * nfeat * 128 + k * 128 + ((((r63 >> 3) ^ (k & 7)) & 7) << 4) + ((r63 & 7) << 1)
            cols.append(base.view(-1, 1) + off + o)
        idx = torch.cat(cols, 1)
        h16.append(recs[idx].int() | (recs[idx + 1].int() << 8))
        words = [(lay * 128 + r) * 8 + w for lay in range(9) for w in range(8)]
        widx = base.view(-1, 1) + REC_MASK + 4 * torch.cat(words, 1)
        masks.append(sum(recs[widx + b].long() << (8 * b) for b in range(4)))
    return torch.cat(h16, 0), torch.cat(masks, 0)


def row_frames(c, fi):
    """The frame of every row record_rows returns."""
    per = [fi.view(-1, 1).expand(c.n, c.nc).reshape(-1)]
    if c.nf:
        per.append(fi.view(-1, 1).expand(c.n, c.nc + c.nf).reshape(-1))
    return torch.cat(per).to(c.ro.device)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("nc,nf", [(64, 128), (128, 256), (3, 7), (64, 0)])
def test_forward_equals_single_frame_calls(E, prec, train, nc, nf):
    c = make_case(E, two_iter_rays(E), nc, nf, prec, seed=nc + nf, dir_z=True)
    ex, la = frames(E, F)
    fi = frame_index(c.n, F)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    multi = {k: v.clone() for k, v in render(E, c, train, fi).items() if k in OUTS}
    torch.cuda.synchronize()
    if train:  # the saved records too, row by row: activations, encodings and ReLU masks of every sample row
        rec_multi = record_rows(E, c)
        rf = row_frames(c, fi)
    for f in range(F):
        E.eng.set_frame(ex[f], la[f])
        one = render(E, c, train)
        sel = (fi == f).to(E.dev)
        for k in multi:
            assert torch.equal(multi[k][sel], one[k][sel]), (f, k)
        if train:
            rec_one = record_rows(E, c)
            rs = rf == f
            assert torch.equal(rec_multi[0][rs], rec_one[0][rs]) and torch.equal(rec_multi[1][rs], rec_one[1][rs]), f
    assert all(torch.isfinite(v).all() for v in multi.values())


def split_case(c, idx, ex, la):
    """The rays idx of case c as a single-frame case of frame (ex, la)."""
    s = lambda t: None if t is None else t[idx].contiguous()  # noqa: E731
    return types.SimpleNamespace(n=len(idx), nc=c.nc, nf=c.nf, prec=c.prec, perturb=c.perturb, noise_std=c.noise_std, white=c.white,
                                 noise={k: s(v) for k, v in c.noise.items()}, ro=s(c.ro), rd=s(c.rd), bg=s(c.bg), dz=s(c.dz),
                                 expr=ex, latent=la, mc=c.mc, mf=c.mf)


def multi_backward(E, c, fi, nfr, gouts, want_params=True):
    pc, pf = params_of(c)
    inputs = ["ray_origins", "ray_directions", "expression"] + (["background"] if c.bg is not None else []) + \
        (["dir_z"] if c.dz is not None else [])
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=want_params, inputs=inputs, frames=True)
    torch.cuda.synchronize()
    return gc, gf, gl, ing


def reference_frames(E, c, fi, nfr, ex, la, z_c, z_f, gouts):
    """float64: per frame on that frame's rays; parameters summed over frames, inputs scattered back to their rays."""
    gc = gf = None
    glat = torch.zeros(nfr, 32, dtype=torch.float64, device=E.dev)
    gexp = torch.zeros(nfr, 76, dtype=torch.float64, device=E.dev)
    ins = {}
    for f in range(nfr):
        idx = torch.nonzero(fi.to(E.dev) == f).flatten()
        if len(idx) == 0:
            continue
        cf = split_case(c, idx, ex[f], la[f])
        ref, R = reference_inputs(E, cf, z_c[idx], z_f[idx] if z_f is not None else None, [g[idx] if g is not None else None for g in gouts])
        glat[f], gexp[f] = R.glat.reshape(32), ref.pop("expression").reshape(76)
        gc = R.gc if gc is None else [a + b if a is not None else None for a, b in zip(gc, R.gc)]
        if R.gf is not None:
            gf = R.gf if gf is None else [a + b if a is not None else None for a, b in zip(gf, R.gf)]
        for k, v in ref.items():
            if k not in ins:
                ins[k] = torch.zeros((c.n,) + tuple(v.shape[1:]), dtype=torch.float64, device=E.dev)
            ins[k][idx] = v
    return gc, gf, glat, gexp, ins


def param_pairs(gc, gf, rc, rf):
    out = []
    for net, gs, rs in (("coarse", gc, rc), ("fine", gf, rf)):
        if gs is None:
            continue
        out += [(f"{net}.{TR.PARAM_ORDER[i]}", g, r) for i, (g, r) in enumerate(zip(gs, rs)) if g is not None]
    return out


def backward_case(E, c, nfr, want_params=True, seed=0):
    ex, la = frames(E, nfr, seed)
    fi = frame_index(c.n, nfr, seed, empty=EMPTY if nfr > EMPTY else -1)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    s = saved_state(E, c)
    gouts = out_grads(E, c)
    kg = multi_backward(E, c, fi, nfr, gouts, want_params)
    ref = reference_frames(E, c, fi, nfr, ex, la, s.z_c, s.z_f, gouts)
    return fi, ex, la, gouts, kg, ref


def check_backward(c, nfr, kg, ref, tag, want_params=True):
    gc, gf, gl, ing = kg
    rc, rf, rlat, rexp, rins = ref
    if want_params:
        check(f"{tag} params", param_pairs(gc, gf, rc, rf), TOL[c.prec])
    used = [f for f in range(nfr) if float(rlat[f].abs().sum()) > 0]
    check(f"{tag} latent", [(f"latent{f}", gl[f], rlat[f]) for f in used], TOL[c.prec])
    check(f"{tag} expression", [(f"expr{f}", ing["expression"][f], rexp[f]) for f in used], IN_TOL[c.prec])
    check(f"{tag} inputs", [(k, ing[k], rins[k]) for k in rins], IN_TOL[c.prec])
    if nfr > EMPTY:
        assert torch.count_nonzero(gl[EMPTY]) == 0 and torch.count_nonzero(ing["expression"][EMPTY]) == 0


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("mode", ["full", "input_only"])
def test_backward_against_float64(E, prec, mode):
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=11, dir_z=True)
    _, _, _, _, kg, ref = backward_case(E, c, F, want_params=mode == "full")
    check_backward(c, F, kg, ref, f"{prec} {mode}", want_params=mode == "full")


@pytest.mark.parametrize("prec", PRECS)
def test_production_batch_eight_frames(E, prec):
    c = make_case(E, 2048, 64, 64, prec, stress=False, seed=12)
    _, _, _, _, kg, ref = backward_case(E, c, 8, seed=1)
    check_backward(c, 8, kg, ref, f"2048r {prec}")


@pytest.mark.parametrize("prec", PRECS)
def test_chunked_backward_and_reproducible(E, prec, monkeypatch):
    """Over a 48 MiB budget the backward re-runs the multi-frame forward per chunk (frame index advanced with the rays); the
    per-frame sums add in chunk order.  Two identical runs are bit-identical."""
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=19, dir_z=True)
    ex, la = frames(E, F, 2)
    fi = frame_index(c.n, F, 2).to(E.dev)  # the chunked backward re-reads it: it must stay alive, like the rays
    runs = []
    for _ in range(2):
        E.eng.sync_weights(c.mc, c.mf)
        E.eng.set_frames(ex, la)
        l0 = E.eng.launch_count()
        outs = {k: v.clone() for k, v in render(E, c, True, fi).items() if k in OUTS}
        gouts = out_grads(E, c)
        runs.append((outs, multi_backward(E, c, fi, F, gouts)))
        # 48 MiB = 32 rays per chunk: a SAVE forward and at least six backward launches per chunk, so the call was chunked
        assert E.eng.launch_count() - l0 > 7 * (c.n // 32)
    (o1, k1), (o2, k2) = runs
    assert all(torch.equal(o1[k], o2[k]) for k in o1)
    for a, b in zip(list(k1[0]) + list(k1[1]) + [k1[2]], list(k2[0]) + list(k2[1]) + [k2[2]]):
        assert (a is None and b is None) or torch.equal(a, b)
    assert all(torch.equal(k1[3][k], k2[3][k]) for k in k1[3])
    # the one-launch backward of the same forward: per-ray gradients within 1e-3 of it (test_input_grads_gpu.py's chunked bound);
    # parameters, latents and expressions also against float64 (depths from the one-launch forward)
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    s = saved_state(E, c)
    one = multi_backward(E, c, fi, F, gouts)
    for k in one[3]:
        em, el = errors(k1[3][k], one[3][k])
        assert em <= 1e-3 and el <= 1e-3, (k, em, el)
    rc, rf, rlat, rexp, _ = reference_frames(E, c, fi, F, ex, la, s.z_c, s.z_f, gouts)
    check(f"chunked {prec} params", param_pairs(k1[0], k1[1], rc, rf), TOL[prec])
    used = [f for f in range(F) if f != EMPTY]
    check(f"chunked {prec} latent", [(f"latent{f}", k1[2][f], rlat[f]) for f in used], TOL[prec])
    check(f"chunked {prec} expression", [(f"expr{f}", k1[3]["expression"][f], rexp[f]) for f in used], IN_TOL[prec])
    assert torch.count_nonzero(k1[2][EMPTY]) == 0 and torch.count_nonzero(k1[3]["expression"][EMPTY]) == 0


def test_out_of_range_frame_gives_nan_for_those_rays_only(E):
    c = make_case(E, two_iter_rays(E), 64, 64, "fast", seed=4)
    ex, la = frames(E, F)
    fi = frame_index(c.n, F)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    good = {k: v.clone() for k, v in render(E, c, False, fi).items() if k in OUTS}
    bad_fi = fi.clone()
    bad_fi[3], bad_fi[10] = -1, F
    bad = render(E, c, False, bad_fi)
    sel = torch.zeros(c.n, dtype=torch.bool, device=E.dev)
    sel[3] = sel[10] = True
    for k in good:
        assert torch.isnan(bad[k][sel]).all(), k
        assert torch.equal(bad[k][~sel], good[k][~sel]), k


def test_errors(E):
    c = make_case(E, 64, 64, 64, "fast", seed=4)
    cap, lib, h = E.capi, E.capi.lib, E.eng._h
    ex, la = frames(E, F)
    E.eng.sync_weights(c.mc, c.mf)
    big = torch.zeros(cap.NFB_MAX_FRAMES + 1, 108, device=E.dev)
    assert lib.nfb_set_frames(h, big.data_ptr(), big.data_ptr(), cap.NFB_MAX_FRAMES + 1, None) == 2  # UNSUPPORTED
    E.eng.set_frames(ex, la)
    # in-kernel rays (o == NULL) in a multi-frame call
    rays = cap.NfbRays()
    rays.n_rays, rays.height, rays.width, rays.near_, rays.far_ = 64, 8, 8, NEAR, FAR
    rays.pose[0] = rays.pose[5] = rays.pose[10] = 1.0
    rays.intrinsics[0] = rays.intrinsics[1] = 10.0
    sm = cap.NfbSampling(64, 64, 0, 0.0, 0, 0, 0, None, None)
    out = {k: torch.empty((64, 3) if k.startswith("rgb") else (64,), device=E.dev) for k in OUTS}
    o = cap.NfbOutputs(*[out[k].data_ptr() for k in OUTS])
    fi = torch.zeros(64, dtype=torch.int32, device=E.dev)
    assert lib.nfb_render_forward_frames(h, C.byref(rays), fi.data_ptr(), C.byref(sm), None, C.byref(o), None) == 2
    # a multi-frame backward after a single-frame training forward
    E.eng.set_frame(ex[0], la[0])
    render(E, c, True)
    pc, pf = params_of(c)
    with pytest.raises(RuntimeError, match="multi-frame training forward"):
        E.eng.backward(list(out_grads(E, c)), pc, pf, frames=True)
    # single-frame backward asked for the latent after a multi-frame forward
    render(E, c, True, frame_index(c.n, F))
    pc, pf = params_of(c)
    with pytest.raises(RuntimeError):
        E.eng.backward(list(out_grads(E, c)), pc, pf)
    with pytest.raises(RuntimeError):
        E.eng.backward(list(out_grads(E, c)), pc, pf, want_latent=False, want_params=False, inputs=["expression"])


def test_render_and_set_frame_in_between_do_not_change_gradients(E):
    c = make_case(E, two_iter_rays(E), 64, 64, "exact", seed=6)
    ex, la = frames(E, F)
    fi = frame_index(c.n, F)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    gouts = out_grads(E, c)
    k1 = multi_backward(E, c, fi, F, gouts)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    E.eng.set_frame(ex[0] * 2, la[0] * 2)
    E.eng.set_frames(ex.flip(0) * 3, la.flip(0))
    c2 = make_case(E, 100, 32, 16, "fast", seed=7)
    render(E, c2, False)
    k2 = multi_backward(E, c, fi, F, gouts)
    for a, b in zip(list(k1[0]) + list(k1[1]) + [k1[2]], list(k2[0]) + list(k2[1]) + [k2[2]]):
        assert (a is None and b is None) or torch.equal(a, b)
    assert all(torch.equal(k1[3][k], k2[3][k]) for k in k1[3])


def test_dropin_fit_shared_latent_and_expressions(E):
    """Fit one shared latent code plus per-frame expressions to 4 frames with nerf.render_frames + loss.backward() +
    torch.optim.Adam; the gradients of one step equal those of the sum of per-frame single-frame renders."""
    nerf = E.nerf
    c = make_case(E, 512, 32, 32, "exact", seed=9, perturb=False, noise_std=0.0, bg=False)
    for p in list(c.mc.parameters()) + list(c.mf.parameters()):
        p.requires_grad_(False)
    opts = types.SimpleNamespace(
        dataset=types.SimpleNamespace(no_ndc=True, near=NEAR, far=FAR),
        nerf=types.SimpleNamespace(train=types.SimpleNamespace(num_coarse=32, num_fine=32, perturb=False, lindisp=False,
                                                               radiance_field_noise_std=0.0, white_background=False, chunksize=512)))
    nfr = 4
    ex_t, la_t = frames(E, nfr, 3)
    fi = (torch.arange(c.n) % nfr).to(E.dev)
    with torch.no_grad():
        target = nerf.render_frames(c.ro, c.rd, fi, ex_t, la_t.mean(0, keepdim=True).expand(nfr, 32), c.mc, c.mf, opts)[3].clone()
    latent = torch.zeros(1, 32, device=E.dev, requires_grad=True)
    expr = (ex_t + 0.3).clone().requires_grad_(True)
    ids = torch.zeros(nfr, dtype=torch.long, device=E.dev)

    def loss_fn():
        out = nerf.render_frames(c.ro, c.rd, fi, expr, latent[ids], c.mc, c.mf, opts)
        return torch.nn.functional.mse_loss(out[3], target) + torch.nn.functional.mse_loss(out[0], target)

    loss = loss_fn()
    loss.backward()
    g_lat, g_expr = latent.grad.clone(), expr.grad.clone()
    latent.grad = expr.grad = None
    # the same loss as a sum over frames of single-frame renders
    total = 0.0
    for f in range(nfr):
        sel = fi == f
        o = nerf.run_one_iter_of_nerf(48, 48, 1.0, c.mc, c.mf, c.ro[sel], c.rd[sel], opts, "train", expressions=expr[f],
                                      latent_code=latent[0])
        ls = torch.nn.functional.mse_loss(o[3], target[sel], reduction="sum") + torch.nn.functional.mse_loss(o[0], target[sel], reduction="sum")
        ls = ls / (3 * c.n)
        ls.backward()
        total += float(ls.detach())
    check("dropin", [("latent", g_lat, latent.grad), ("expr", g_expr, expr.grad)], (2e-3, 2e-3))
    assert abs(total - float(loss)) <= 1e-5 * abs(total) + 1e-9
    opt = torch.optim.Adam([latent, expr], lr=1e-2)
    first = None
    for _ in range(30):
        opt.zero_grad()
        ls = loss_fn()
        ls.backward()
        opt.step()
        first = float(ls) if first is None else first
    assert float(loss_fn()) < 0.7 * first
