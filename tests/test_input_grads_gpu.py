"""Input gradients of the fused backward (nfb_render_backward_ex: rays, dir_z, background, expression) against a float64
reference, and the drop-in surface that uses them to fit a frozen avatar to images.

The reference is tests/torch_reference.render_at_depths in float64 on the GPU at the depths the kernel sampled, with the
rays, expression, background and dir_z as leaves (the helpers of test_backward_fp64_gpu.py).  Per tensor:
  max |got - ref| <= tol_max * max |ref|,   |got - ref|_2 <= tol_l2 * |ref|_2
Tolerances (IN_TOL) come from measurements on an H100 80GB HBM3 (CUDA 12.9), recorded beside them.  The gradients with
respect to a point are sums of 63 PE columns, the high frequencies scaled by up to 2^9, of FP16 dY rows; in fast mode the
forward's saved state carries FP16 rounding as well, which is why fast mode has the wider bounds."""
import types

import pytest
import torch

import torch_reference as TR
from test_backward_fp64_gpu import (E, FAR, NEAR, PRECS, TOL, check, errors, grad_pairs, make_case, out_grads,  # noqa: F401
                                    saved_state, train_forward, two_iter_rays)

pytestmark = pytest.mark.gpu

# (max, L2) per input-gradient tensor.  Measured worst over all cases (H100 80GB HBM3, 400 W):
#   exact: max 9.2e-3 (ray_origins, dir_z case), L2 2.6e-3      fast: max 7.2e-2 (ray_origins, 100c+60f), L2 4.8e-2 (64c+0f)
IN_TOL = {"exact": (2e-2, 6e-3), "fast": (1.5e-1, 1e-1)}
ALONE_TOL = {"exact": (6e-2, 1.5e-2)}  # one output gradient alone: measured max 2.9e-2, L2 5.3e-3 (rgb_fine alone, ray_origins)
ACC_NOISE_IN = 1e-4  # acc-only input gradients relative to the rgb-only ones of the same pass (both are rounding noise; below)


def wanted(c):
    return ["ray_origins", "ray_directions", "expression"] + (["background"] if c.bg is not None else []) + \
        (["dir_z"] if c.dz is not None else [])


def params_of(c):
    pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
    pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER] if c.mf is not None else None
    return pc, pf


def kernel_inputs(E, c, gouts, want_params=False):
    pc, pf = params_of(c)
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=want_params, inputs=wanted(c))
    torch.cuda.synchronize()
    return (gc, gf, gl), ing


def reference_inputs(E, c, z_c, z_f, gouts):
    """float64 gradients of sum_i <out_i, gouts_i> with respect to the inputs, the latent and the parameters."""
    f64 = lambda t: None if t is None else t.detach().to(E.dev, torch.float64)  # noqa: E731
    leaf = lambda t: None if t is None else f64(t).requires_grad_(True)  # noqa: E731
    pc = {k: leaf(v) for k, v in c.mc.named_parameters()}
    pf = {k: leaf(v) for k, v in c.mf.named_parameters()} if c.mf is not None else None
    ro, rd, expr, lat, bg, dz = leaf(c.ro), leaf(c.rd), leaf(c.expr), leaf(c.latent), leaf(c.bg), leaf(c.dz)
    n = c.n
    nearfar = torch.tensor([NEAR, FAR], device=E.dev, dtype=torch.float64).expand(n, 2)
    chunk = max(16, 65536 // (2 * c.nc + c.nf))
    for b in range(0, n, chunk):
        s = slice(b, min(n, b + chunk))
        rays = torch.cat((ro[s], rd[s], nearfar[s]), -1)
        o = TR.render_at_depths(rays, pc, pf, expr, lat, f64(z_c[s]), f64(z_f[s]) if z_f is not None else None, NEAR, FAR,
                                c.noise_std, {k: f64(v[s]) for k, v in c.noise.items()}, c.white,
                                bg[s] if bg is not None else None, dz[s] if dz is not None else None)
        loss = sum(((oi * f64(gi[s])).sum() for oi, gi in zip(o, gouts) if oi is not None and gi is not None),
                   torch.zeros((), dtype=torch.float64, device=E.dev))
        loss.backward()
    ref = dict(ray_origins=ro.grad, ray_directions=rd.grad, expression=expr.grad)
    if bg is not None:
        ref["background"] = bg.grad
    if dz is not None:
        ref["dir_z"] = dz.grad
    return ref, types.SimpleNamespace(gc=[pc[k].grad for k in TR.PARAM_ORDER],
                                      gf=[pf[k].grad for k in TR.PARAM_ORDER] if pf is not None else None, glat=lat.grad)


def kernel_names(prof):
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


def input_pairs(ing, ref):
    return [(k, ing[k], ref[k]) for k in ref]


def run_case(E, c, tag, gouts=None, tol=None):
    train_forward(E, c)
    s = saved_state(E, c)
    gouts = out_grads(E, c) if gouts is None else gouts
    kg, ing = kernel_inputs(E, c, gouts)
    ref, R = reference_inputs(E, c, s.z_c, s.z_f, gouts)
    check(f"{tag} inputs", input_pairs(ing, ref), tol or IN_TOL[c.prec])
    check(f"{tag} latent", [("latent", kg[2], R.glat)], TOL[c.prec])
    return kg, ing, ref, R


@pytest.mark.parametrize("prec", PRECS)
def test_production_batch(E, prec):
    """2048 rays at 64c+64f with perturbation, sigma noise and a background."""
    run_case(E, make_case(E, 2048, 64, 64, prec, stress=False), f"2048r {prec}")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("nc,nf", [(64, 64), (100, 60), (256, 256), (64, 0)])
def test_sample_counts(E, prec, nc, nf):
    """4 SMs + 37 rays (every CTA runs two units, the last unit half filled); 100c+60f and 256c+256f put rays across tiles."""
    run_case(E, make_case(E, two_iter_rays(E), nc, nf, prec, seed=nc + nf), f"{nc}c+{nf}f {prec}")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("opt", ["white", "nobg", "dir_z"])
def test_compositing_options(E, prec, opt):
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=3, bg=opt == "dir_z", white=opt == "white", dir_z=opt == "dir_z")
    run_case(E, c, f"{opt} {prec}")


@pytest.mark.parametrize("which", range(7))
def test_each_output_alone(E, which):
    """disp alone reaches the rays only through the sample spacings (the |d| term) and the density.  acc = 1 - prod(1 - alpha
    + 1e-10) is 1 to within rounding on every ray (the last interval is 1e10 long), so its gradients are rounding noise on both
    sides: they are bounded by the gradients the same-sized rgb output gradient of the same pass makes."""
    c = make_case(E, two_iter_rays(E), 64, 64, "exact", seed=4, dir_z=True)
    if which not in (2, 5):
        run_case(E, c, f"output {which}", gouts=out_grads(E, c, which=which), tol=ALONE_TOL["exact"])
        return
    train_forward(E, c)
    _, ing_acc = kernel_inputs(E, c, out_grads(E, c, which=which))
    _, ing_rgb = kernel_inputs(E, c, out_grads(E, c, which=which - 2))
    for k in ing_acc:
        assert bool(torch.isfinite(ing_acc[k]).all()), k
        noise = float(ing_acc[k].abs().max()) / float(ing_rgb[k].abs().max())
        print(f"only output {which} {k}: max |gradient| / rgb-gradient scale {noise:.2e}")
        assert noise <= ACC_NOISE_IN, (k, noise)


@pytest.mark.parametrize("prec", PRECS)
def test_input_only_matches_full_backward(E, prec):
    """Input-only mode (no parameter gradient) gives the same input gradients and d latent as a full backward on the same
    saved forward, in fewer launches; the full backward's parameter gradients stay within the float64 bounds."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=8, dir_z=True)
    train_forward(E, c)
    s = saved_state(E, c)
    gouts = out_grads(E, c)
    l0 = E.eng.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof_full:
        kg_full, ing_full = kernel_inputs(E, c, gouts, want_params=True)
    l1 = E.eng.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof_in:
        kg_in, ing_in = kernel_inputs(E, c, gouts, want_params=False)
    l2 = E.eng.launch_count()
    assert kg_in[0] is None and kg_in[1] is None
    assert l2 - l1 < l1 - l0, (l1 - l0, l2 - l1)
    # which kernels ran: input-only mode runs the PE-only weight-gradient launch and neither the full one nor finalize
    names_full, names_in = kernel_names(prof_full), kernel_names(prof_in)
    assert any("dw_kernel<false>" in k for k in names_full) and any("finalize_kernel" in k for k in names_full), names_full
    assert any("dw_kernel<true>" in k for k in names_in), names_in
    assert not any("dw_kernel<false>" in k or "finalize_kernel" in k or "fin_dir0_kernel" in k for k in names_in), names_in
    for k in ing_full:
        em, el = errors(ing_in[k], ing_full[k])
        assert em <= 1e-5 and el <= 1e-5, (k, em, el)
    em, el = errors(kg_in[2], kg_full[2])
    assert em <= 1e-5 and el <= 1e-5, ("latent", em, el)
    ref, R = reference_inputs(E, c, s.z_c, s.z_f, gouts)
    check(f"full+inputs {prec} params", grad_pairs(kg_full, R), TOL[prec])
    check(f"full+inputs {prec} inputs", input_pairs(ing_full, ref), IN_TOL[prec])


@pytest.mark.parametrize("prec", PRECS)
def test_chunked_matches_one_launch(E, prec, monkeypatch):
    """Over the memory budget the per-ray gradients are written chunk by chunk and expression / latent add up over chunks."""
    c = make_case(E, two_iter_rays(E), 64, 64, prec, seed=19, dir_z=True)
    train_forward(E, c)
    gouts = out_grads(E, c, seed=20)
    _, one = kernel_inputs(E, c, gouts)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    l0 = E.eng.launch_count()
    train_forward(E, c)
    _, chk = kernel_inputs(E, c, gouts)
    # 48 MiB = 16 units of 3 one-MiB tiles = 32 rays per chunk: a SAVE forward and at least five backward launches per chunk
    assert E.eng.launch_count() - l0 > 6 * (c.n // 32)
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    for k in one:
        em, el = errors(chk[k], one[k])
        print(f"chunked vs one launch {prec} {k}: max {em:.2e}, L2 {el:.2e}")
        assert em <= 1e-3 and el <= 1e-3, (k, em, el)


def test_missing_inputs_are_invalid(E):
    """Background / dir_z gradients without a background / dir_z in the forward are invalid arguments."""
    c = make_case(E, 256, 64, 64, "fast", bg=False)
    train_forward(E, c)
    pc, pf = params_of(c)
    gouts = out_grads(E, c)
    for name in ("background", "dir_z"):
        with pytest.raises(RuntimeError, match="invalid"):
            E.eng.backward(gouts, pc, pf, want_params=False, inputs=[name])


# ------------------------------------------------------------------------------------------------ drop-in surface
def _dropin(E, nerf, stress=True):
    from test_backward_fp64_gpu import model
    mc, mf = model(E, 100, stress), model(E, 101, stress)
    blk = dict(num_coarse=64, num_fine=64, perturb=False, lindisp=False, radiance_field_noise_std=0.0,
               white_background=False, chunksize=2048)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=NEAR, far=FAR)))
    return mc, mf, cfg


def test_dropin_frozen_avatar_expression_and_pose(E):
    """Frozen networks, expression and camera pose require grad: run_one_iter_of_nerf -> MSE -> loss.backward() reaches the
    expression and, through the torch ray bundle, the pose; the networks' .grad stay None."""
    nerf = E.nerf
    import nerface_oracle as O
    mc, mf, cfg = _dropin(E, nerf)
    for m in (mc, mf):
        m.requires_grad_(False)
    fr = O.synthetic_frame(21, 24, 24)
    H = W = 24
    pose = fr["pose"].to(E.dev).clone().requires_grad_(True)
    expr = fr["expr"].to(E.dev).clone().requires_grad_(True)
    lat = fr["latent"].to(E.dev)
    target = torch.rand(H * W, 3, generator=torch.Generator().manual_seed(3)).to(E.dev)
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], pose)
    out = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro.reshape(-1, 3), rd.reshape(-1, 3), cfg, mode="train",
                                    expressions=expr, latent_code=lat)
    loss = ((out[0] - target) ** 2).mean() + ((out[3] - target) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    assert all(p.grad is None for m in (mc, mf) for p in m.parameters())
    s = E.eng.train_debug()
    from test_backward_gpu import dev_tensor
    n = H * W
    z_c = dev_tensor(s.z_coarse, (n, 64)).clone().double()
    z_f = dev_tensor(s.z_fine, (n, 128)).clone().double()
    # float64 reference through the same torch ray bundle
    p64 = pose.detach().double().requires_grad_(True)
    e64 = expr.detach().double().requires_grad_(True)
    ro64, rd64 = nerf.get_ray_bundle(H, W, fr["intrinsics"], p64)
    ro64, rd64 = ro64.reshape(-1, 3), rd64.reshape(-1, 3)
    pc = {k: v.detach().double() for k, v in mc.named_parameters()}
    pf = {k: v.detach().double() for k, v in mf.named_parameters()}
    nearfar = torch.tensor([NEAR, FAR], device=E.dev, dtype=torch.float64).expand(n, 2)
    o = TR.render_at_depths(torch.cat((ro64, rd64, nearfar), -1), pc, pf, e64, lat.double(), z_c, z_f, NEAR, FAR)
    t64 = target.double()
    ref_loss = ((o[0] - t64) ** 2).mean() + ((o[3] - t64) ** 2).mean()
    ref_loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss.detach())) <= 1e-3 * float(ref_loss.detach())
    check("drop-in expression", [("expression", expr.grad, e64.grad)], IN_TOL["fast"])
    check("drop-in pose", [("pose", pose.grad[:3], p64.grad[:3])], IN_TOL["fast"])


def test_dropin_fit_expression_lowers_loss(E):
    """A short deterministic fit: render a target at one expression, start from a perturbed one, 30 Adam steps on the
    expression alone (frozen stress-weight networks) lower the photometric loss."""
    nerf = E.nerf
    import nerface_oracle as O
    mc, mf, cfg = _dropin(E, nerf)
    for m in (mc, mf):
        m.requires_grad_(False)
    fr = O.synthetic_frame(21, 16, 16)
    H = W = 16
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(E.dev))
    ro, rd = ro.reshape(-1, 3).contiguous(), rd.reshape(-1, 3).contiguous()
    lat = fr["latent"].to(E.dev)
    true_expr = fr["expr"].to(E.dev)
    with torch.no_grad():
        tgt = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="train", expressions=true_expr,
                                        latent_code=lat)[3].clone()
    g = torch.Generator().manual_seed(9)
    expr = (true_expr + 0.5 * torch.randn(76, generator=g).to(E.dev)).requires_grad_(True)
    opt = torch.optim.Adam([expr], lr=2e-2)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        out = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="train", expressions=expr,
                                        latent_code=lat)
        loss = ((out[3] - tgt) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print("fit losses", losses[0], losses[-1])
    assert losses[-1] < 0.5 * losses[0], losses


def test_ray_gradients_after_in_kernel_rays_are_unsupported(E):
    """A training forward that generated its rays in the kernel (NfbRays.o == NULL) has no ray tensors to differentiate: ray
    gradients are NFB_ERR_UNSUPPORTED, while the expression gradient of the same backward is still available."""
    import ctypes as C
    capi = E.capi
    c = make_case(E, 64, 64, 64, "fast", bg=False)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frame(c.expr, c.latent)
    H = W = 8
    n = H * W
    out = torch.empty(11, n, device=E.dev)
    rays = capi.NfbRays()
    rays.n_rays = n
    pose = torch.eye(4)[:3].reshape(-1)
    pose[11] = 1.5
    for i in range(12):
        rays.pose[i] = float(pose[i])
    for i, v in enumerate((12.0, 12.0, 0.5, 0.5)):
        rays.intrinsics[i] = v
    rays.height, rays.width, rays.row_begin, rays.near_, rays.far_ = H, W, 0, NEAR, FAR
    sm = capi.NfbSampling(64, 64, 0, 0.0, 0, 0, capi.NFB_PREC_FAST, None, None)
    f = out.view(-1)
    o = capi.NfbOutputs(*[f[k * n:].data_ptr() for k in (0, 3, 4, 5, 8, 9, 10)])
    assert capi.lib.nfb_render_forward_train(E.eng._h, C.byref(rays), C.byref(sm), None, C.byref(o), None) == 0
    E.eng.train_rays = n
    pc, pf = params_of(c)
    gouts = [torch.ones(n, 3, device=E.dev) / n, None, None, torch.ones(n, 3, device=E.dev) / n, None, None, None]
    for name in ("ray_origins", "ray_directions"):
        with pytest.raises(RuntimeError, match="not supported"):
            E.eng.backward(gouts, pc, pf, want_params=False, inputs=[name])
    _, _, gl, ing = E.eng.backward(gouts, pc, pf, want_params=False, inputs=["expression"])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(ing["expression"]).all()) and float(ing["expression"].abs().max()) > 0


def test_dropin_ablation_directions(E):
    """ray_directions_ablation requiring grad through run_one_iter_of_nerf: every chunk's direction encoder reads chunk 0 of
    the ablation bundle (train_utils.py:81-82), so chunk 0's z column receives the sum over chunks, as in the reference."""
    nerf = E.nerf
    import nerface_oracle as O
    mc, mf, cfg = _dropin(E, nerf)
    cfg.nerf.train.chunksize = 128
    for m in (mc, mf):
        m.requires_grad_(False)
    H = W = 16
    n = H * W
    fr, fr2 = O.synthetic_frame(21, H, W), O.synthetic_frame(22, H, W)
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(E.dev))
    abl = nerf.get_ray_bundle(H, W, fr2["intrinsics"], fr2["pose"].to(E.dev))[1].reshape(-1, 3).contiguous().requires_grad_(True)
    ro, rd = ro.reshape(-1, 3).contiguous(), rd.reshape(-1, 3).contiguous()
    lat = fr["latent"].to(E.dev)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(4)).to(E.dev)
    out = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="train", expressions=fr["expr"].to(E.dev),
                                    latent_code=lat, ray_directions_ablation=abl)
    loss = ((out[0] - target) ** 2).mean() + ((out[3] - target) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    s = E.eng.train_debug()
    from test_backward_gpu import dev_tensor
    z_c = dev_tensor(s.z_coarse, (n, 64)).clone().double()
    z_f = dev_tensor(s.z_fine, (n, 128)).clone().double()
    a64 = abl.detach().double().requires_grad_(True)
    dz = torch.cat([a64[:128, 2]] * (n // 128))
    pc = {k: v.detach().double() for k, v in mc.named_parameters()}
    pf = {k: v.detach().double() for k, v in mf.named_parameters()}
    nearfar = torch.tensor([NEAR, FAR], device=E.dev, dtype=torch.float64).expand(n, 2)
    o = TR.render_at_depths(torch.cat((ro.double(), rd.double(), nearfar), -1), pc, pf, fr["expr"].to(E.dev).double(), lat.double(),
                            z_c, z_f, NEAR, FAR, dir_z=dz)
    t64 = target.double()
    (((o[0] - t64) ** 2).mean() + ((o[3] - t64) ** 2).mean()).backward()
    assert float(abl.grad[128:].abs().max()) == 0.0 and float(abl.grad[:, :2].abs().max()) == 0.0
    check("drop-in ablation", [("ray_directions_ablation", abl.grad, a64.grad)], IN_TOL["fast"])
