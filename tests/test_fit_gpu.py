"""Fitting steps over several images (NFB_FIT_STEP): nfb_fit_rows_grad against its documented FP32 order and float64,
nerf.FusedFitter's gradients against torch autograd through rays rebuilt from a requires_grad pose, its step against
torch.optim.Adam with three parameter groups, frozen tables and networks, the aliasing of the sampler's tables, the captured
step against the eager one, the step over the memory budget, and the launches per step."""
import re

import numpy as np
import pytest
import torch

import nerface_oracle as O
from test_backward_gpu import dev_tensor
from test_fit_cpu import camera_dirs, gamma, pose_rows_fp32, slot_terms

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train, ray_sampler
    return nerf, _engine, fused_train, ray_sampler, torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def own_renderer(env, monkeypatch):
    """A renderer handle of the test's own: its buffers start empty, and an exact-grad fit (which adds the lo-stream launch to
    every later re-pack on its handle) leaves the handle other test files count launches on alone."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.Renderer(dev)
    monkeypatch.setitem(_engine._renderers, ("cuda", dev.index), eng)
    yield eng
    torch.cuda.synchronize()


def make_model(nerf, params, dev):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params)
    return m.to(dev).requires_grad_(False)


def frames(n_images, H, seed=0):
    frs = [O.synthetic_frame(seed + i, H, H) for i in range(n_images)]
    g = torch.Generator().manual_seed(seed + 100)
    images = torch.rand(n_images, H, H, 3, generator=g)
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs])
    lats = torch.randn(n_images, 32, generator=g) * 0.1
    return frs, images, poses, exprs, lats


BOXES = [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20), (0, 32, 0, 32), (12, 20, 12, 20), (2, 28, 4, 16), (6, 26, 6, 26),
         (1, 31, 3, 29)]


def fitter(env, n_images=6, H=32, background=True, seed=0, **kw):
    nerf, _engine, fused_train, ray_sampler, dev = env
    frs, images, poses, exprs, lats = frames(n_images, H, seed)
    opts = dict(num_coarse=64, num_fine=64, perturb=True, noise_std=0.1)
    opts.update(kw)
    return nerf.FusedFitter(make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev),
                            images.to(dev), BOXES[:n_images], frs[0]["intrinsics"], poses, exprs, lats,
                            background=frs[0]["bg"].to(dev) if background else None, **opts)


def draws_for(dev, k, n, rounds, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=g)


# ---------------------------------------------------------------------------------------------------------------- 1. the rows
@pytest.mark.parametrize("K,n,H,case", [(1, 1, 32, "plain"), (3, 777, 64, "plain"), (64, 2048, 64, "plain"), (6, 300, 64, "repeats"),
                                        (4, 200, 64, "out_of_range"), (2, 2048, 64, "short"), (3, 500, 64, "nan"),
                                        (3, 256, 64, "null")])
def test_rows_follow_their_definition(env, K, n, H, case):
    """Pose and expression rows bit for bit the documented FP32 order (tests/test_fit_cpu.py restates it) and within
    gamma(n + K + 2) * sum|term| of float64; the camera directions are the sampler's bits (an identity rotation makes the rays'
    x, y components exactly cx, cy)."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    n_img = 5
    frs, images, poses, exprs, lats = frames(n_img, H, seed=3)
    poses[0] = torch.tensor([1.0, 0, 0, 0.1, 0, 1.0, 0, -0.2, 0, 0, 1.0, 0.7])  # identity rotation
    boxes = [(4, H - 4, 2, H - 8), (0, H, 0, H), (10, 30, 12, 40), (2, 3, 2, 4) if case == "short" else (5, 40, 5, 40), (0, 20, 0, 60)]
    data = ray_sampler.TrainImages(images.to(dev), poses, exprs, boxes, frs[0]["intrinsics"], device=dev)
    rng = np.random.default_rng(K * 7 + n)
    img = [int(v) for v in rng.integers(0, n_img, K)]
    img[0] = 0
    if case == "repeats":
        img = [2, 0, 2, 2, 1, 0]
    if case == "short":
        img = [3, 0]
    rounds = 1 if case == "short" else 16
    draws = draws_for(dev, K, n, rounds, 11)
    N = K * n
    sb = dict(ray_origins=torch.empty(N, 3, device=dev), ray_directions=torch.empty(N, 3, device=dev),
              pixel_rc=torch.empty(N, 2, dtype=torch.int32, device=dev), state=torch.empty(K, 3, dtype=torch.int32, device=dev))
    idx = torch.tensor(img, dtype=torch.int32, device=dev)
    eng.sample_images(data, idx, n, draws, rounds, torch.zeros(n_img, 32, device=dev), sb)
    if case == "short":
        assert int(sb["state"][0, 0]) < n
    sampled = list(img)
    if case == "out_of_range":
        img = [img[0], n_img, -1, img[3]]
        idx = torch.tensor(img, dtype=torch.int32, device=dev)
    g = torch.Generator().manual_seed(K + n)
    scale = 10.0 ** torch.randint(-6, 1, (N, 1), generator=g).float()
    go = torch.randn(N, 3, generator=g) * scale
    gd = torch.randn(N, 3, generator=g) * scale
    if case == "nan":
        gd[n + 17, 1] = float("nan")
        go[n + 3, 2] = float("nan")
    gexpr = torch.randn(K, 76, generator=g)
    P0 = torch.randn(n_img, 12, generator=g)
    E0 = torch.randn(n_img, 76, generator=g)
    P, E = P0.clone().to(dev), E0.clone().to(dev)
    if case == "null":
        eng.fit_rows_grad(data, idx, n, sb["pixel_rc"], go.to(dev), gd.to(dev), None, None, None)
        eng.fit_rows_grad(data, idx, n, sb["pixel_rc"], None, None, None, gexpr.to(dev), E)
        torch.cuda.synchronize()
        assert torch.equal(P.cpu(), P0)
        _, want_e, _ = pose_rows_fp32(img, n, n_img, sb["pixel_rc"].cpu().numpy(), None, gd.numpy(), data.intrinsics, H, H,
                                      P0.numpy(), gexpr.numpy(), E0.numpy())
        assert np.array_equal(E.cpu().numpy(), want_e)
        eng.fit_rows_grad(data, idx, n, sb["pixel_rc"], go.to(dev), None, P, None, None)  # origins only: the R columns stay
        torch.cuda.synchronize()
        assert torch.equal(P.cpu().view(n_img, 3, 4)[:, :, :3], P0.view(n_img, 3, 4)[:, :, :3])
        return
    eng.fit_rows_grad(data, idx, n, sb["pixel_rc"], go.to(dev), gd.to(dev), P, gexpr.to(dev), E)
    torch.cuda.synchronize()
    rc = sb["pixel_rc"].cpu().numpy()
    want_p, want_e, slots = pose_rows_fp32(img, n, n_img, rc, go.numpy(), gd.numpy(), data.intrinsics, H, H, P0.numpy(), gexpr.numpy(),
                                           E0.numpy())
    got_p, got_e = P.cpu().numpy(), E.cpu().numpy()
    assert np.array_equal(got_p, want_p, equal_nan=True)
    assert np.array_equal(got_e, want_e, equal_nan=True)
    # the camera directions: image 0 has an identity rotation, so the sampler's d = (cx, cy, -1) exactly on its slots
    fx, fy = data.intrinsics[0], data.intrinsics[1]
    cx, cy = camera_dirs(rc, fx, fy, np.float32(H * data.intrinsics[2]), np.float32(H * data.intrinsics[3]))
    rd = sb["ray_directions"].cpu().numpy()
    zero = [k for k in range(K) if sampled[k] == 0]
    assert zero
    for k in zero:
        s = slice(k * n, (k + 1) * n)
        assert np.array_equal(rd[s, 0], cx[s]) and np.array_equal(rd[s, 1], cy[s])
    # float64
    terms = slot_terms(cx, cy, go.numpy(), gd.numpy()).astype(np.float64)
    for r in range(n_img):
        ks = [k for k in range(K) if img[k] == r]
        t = np.concatenate([terms[k * n:(k + 1) * n] for k in ks] + [np.zeros((0, 12))])
        want = P0[r].double().numpy() + t.sum(0)
        bound = gamma(n + K + 2) * (np.abs(P0[r].double().numpy()) + np.abs(t).sum(0))
        finite = ~np.isnan(want)
        assert np.array_equal(np.isnan(got_p[r]), ~finite), r
        assert (np.abs(got_p[r][finite] - want[finite]) <= bound[finite]).all(), r
        if not ks:
            assert np.array_equal(got_p[r], P0[r].numpy()) and np.array_equal(got_e[r], E0[r].numpy())
    if case == "nan":  # only slot 1's image row holds NaN, and only in the columns of the NaN components
        for r in range(n_img):
            assert np.isnan(got_p[r]).any() == (r == img[1]), r
        assert set(np.flatnonzero(np.isnan(got_p[img[1]]))) == {4, 5, 6, 11}


# ------------------------------------------------------------------------------------------------- 2. gradients vs autograd
def torch_rays(data, pose_slots, pixel_rc, k, n):
    """The sampler's rays rebuilt in torch from per-slot [K,12] poses at pixel_rc, the FP32 operation order of get_ray_bundle /
    the sampler (tensor / tensor divisions round once: no reciprocal)."""
    dev = pose_slots.device
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)  # noqa: E731
    fx, fy = f32(data.intrinsics[0]), f32(data.intrinsics[1])
    wcx, hcy = f32(float(data.W) * data.intrinsics[2]), f32(float(data.H) * data.intrinsics[3])
    rc = pixel_rc.long()
    cx = (rc[:, 1].float() - wcx) / fx
    cy = -((rc[:, 0].float() - hcy) / fy)
    P = pose_slots.view(k, 3, 4).repeat_interleave(n, dim=0)
    rd = torch.stack([cx * P[:, q, 0] + cy * P[:, q, 1] + (-1.0) * P[:, q, 2] for q in range(3)], dim=1)
    ro = P[:, :, 3]
    return ro, rd


def cfg_for(nerf, perturb=True, noise=0.1, chunk=1 << 20):
    blk = dict(num_coarse=64, num_fine=64, perturb=perturb, lindisp=False, radiance_field_noise_std=noise, white_background=False,
               chunksize=chunk)
    return nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))


@pytest.mark.parametrize("ids", [[3], [0, 1], [2, 0, 2, 1], [0, 1, 2, 3, 4, 5, 6, 7]])
@pytest.mark.parametrize("precision", ["fast", "exact", "exact_grad"])
@pytest.mark.parametrize("bg", [True, False])
def test_gradients_match_autograd(env, ids, precision, bg):
    """FusedFitter.gradients against nerf.render_frames + MSE + MSE on rays rebuilt in torch from requires_grad per-slot poses
    (equal to the sampler's rays bit for bit) and per-slot expression / latent leaves, the same noise: expression and latent rows
    bitwise the slot gradients for distinct indices and within gamma(K) * sum|.| of their sum with repeats (same kernels, other
    routing); pose rows within 2 gamma(n K + 2) * sum|term| of torch's reduction over the same per-ray gradients."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    k, n = len(ids), 64
    fit = fitter(env, n_images=8, background=bg, precision=precision, latent_reg=0.0)
    draws = draws_for(dev, k, n, 16, 5)
    torch.manual_seed(21)
    loss = fit.gradients(ids, n, draws=draws, max_rounds=16).clone()
    torch.cuda.synchronize()
    sb = fit._last
    ids_t = torch.tensor(ids, device=dev)
    pose = fit.poses[ids_t].clone().requires_grad_(True)
    expr = fit.expressions[ids_t].clone().requires_grad_(True)
    lat = fit.latents[ids_t].clone().requires_grad_(True)
    ro, rd = torch_rays(fit.data, pose, sb["pixel_rc"], k, n)
    assert torch.equal(ro.detach(), sb["ray_origins"]) and torch.equal(rd.detach(), sb["ray_directions"])
    _engine.set_precision(precision)
    try:
        torch.manual_seed(21)
        out = nerf.render_frames(ro, rd, sb["frame_index"], expr, lat, fit.mc, fit.mf, cfg_for(nerf), mode="train",
                                 background_prior=sb["background"] if bg else None)
        coarse = torch.nn.functional.mse_loss(out[0], sb["target"])
        fine = torch.nn.functional.mse_loss(out[3], sb["target"])
        (coarse + fine).backward()
    finally:
        _engine.set_precision("fast")
    assert abs(float(coarse) - float(loss[0])) <= 1e-6 * float(coarse) and abs(float(fine) - float(loss[1])) <= 1e-6 * float(fine)
    ge, gl, gp = (fit._table(fit.grads, t).cpu() for t in ("expression", "latent", "pose"))
    for r in range(8):
        ks = [j for j in range(k) if ids[j] == r]
        for got, leaf in ((ge, expr.grad), (gl, lat.grad)):
            if not ks:
                assert not got[r].any()
            elif len(ks) == 1:
                assert torch.equal(got[r], leaf[ks[0]].cpu()), r
            else:
                want = sum(leaf[j].double().cpu() for j in ks)
                assert ((got[r].double() - want).abs() <= gamma(len(ks)) * sum(leaf[j].double().cpu().abs() for j in ks)).all()
        if ks:
            gro, grd = sb["gro"], sb["grd"]
            rows = torch.cat([torch.arange(j * n, (j + 1) * n) for j in ks])
            rc = sb["pixel_rc"].cpu().numpy()[rows.numpy()]
            cx, cy = camera_dirs(rc, fit.data.intrinsics[0], fit.data.intrinsics[1], np.float32(32 * fit.data.intrinsics[2]),
                                 np.float32(32 * fit.data.intrinsics[3]))
            mag = np.abs(slot_terms(cx, cy, gro.cpu().numpy()[rows.numpy()], grd.cpu().numpy()[rows.numpy()]).astype(np.float64)).sum(0)
            want = sum(pose.grad[j].double().cpu() for j in ks).numpy()
            assert (np.abs(gp[r].double().numpy() - want) <= 2 * gamma(n * len(ks) + 2) * mag + 1e-30).all(), r
        else:
            assert not gp[r].any()


# --------------------------------------------------------------------------------------------- 4. the step vs torch.optim.Adam
def test_step_matches_torch_adam(env):
    """Three parameter groups with their own learning rates, the regulariser on: after one step the tables agree within 7.5e-9
    plus one rounding of the parameter, and the losses within 2e-6 over 10 steps."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    ids, n, rounds, steps = [1, 4, 1, 0], 64, 16, 10
    lrs = dict(lr_pose=2e-4, lr_expression=5e-4, lr_latent=1e-3)
    fit = fitter(env, n_images=6, latent_reg=0.005, **lrs)
    frs, images, poses, exprs, lats = frames(6, 32)
    P = poses.clone().to(dev).requires_grad_(True)
    Ex = exprs.clone().to(dev).requires_grad_(True)
    L = lats.clone().to(dev).requires_grad_(True)
    opt = torch.optim.Adam([dict(params=[P], lr=lrs["lr_pose"]), dict(params=[Ex], lr=lrs["lr_expression"]),
                            dict(params=[L], lr=lrs["lr_latent"])], betas=(0.9, 0.999), eps=1e-8)
    data = ray_sampler.TrainImages(images.to(dev), poses, exprs, BOXES[:6], frs[0]["intrinsics"], background=frs[0]["bg"], device=dev)
    eng = _engine.renderer_for(dev)
    ids_t = torch.tensor(ids, device=dev)
    k = len(ids)
    for i in range(steps):
        draws = draws_for(dev, k, n, rounds, 40 + i)
        torch.manual_seed(500 + i)
        lf = fit.step(ids, n, draws=draws, max_rounds=rounds).clone()
        b = dict(pixel_rc=torch.empty(k * n, 2, dtype=torch.int32, device=dev), target=torch.empty(k * n, 3, device=dev),
                 background=torch.empty(k * n, 3, device=dev), frame_index=torch.empty(k * n, dtype=torch.int32, device=dev))
        eng.sample_images(data, ids_t.int(), n, draws, rounds, L.detach(), b)
        ro, rd = torch_rays(data, P[ids_t], b["pixel_rc"], k, n)
        torch.manual_seed(500 + i)
        out = nerf.render_frames(ro, rd, b["frame_index"], Ex[ids_t], L[ids_t], fit.mc, fit.mf, cfg_for(nerf), mode="train",
                                 background_prior=b["background"])
        coarse = torch.nn.functional.mse_loss(out[0], b["target"])
        fine = torch.nn.functional.mse_loss(out[3], b["target"])
        loss = coarse + fine + (0.005 / k) * sum(torch.norm(L[j]) for j in ids)
        loss.backward()
        opt.step()
        opt.zero_grad()
        if i == 0:  # torch's addcdiv_ rounds the update in another order: one rounding of the parameter may separate the two
            for name, ref in (("poses", P), ("expressions", Ex), ("latents", L)):
                d = (getattr(fit, name) - ref.detach()).abs()
                ulp = torch.from_numpy(np.spacing(ref.detach().abs().cpu().numpy())).to(dev)
                print(f"after one step, {name}: max|fused - torch.optim.Adam| = {float(d.max()):.3e}, "
                      f"beyond one ulp of the parameter {float((d - ulp).max()):.3e}")
                assert bool((d <= 7.5e-9 + ulp).all()), name
        assert abs(float(lf[0]) - float(coarse)) < 2e-6 and abs(float(lf[1]) - float(fine)) < 2e-6, (i, lf, coarse, fine)
    assert fit.iter == steps


# ---------------------------------------------------------------------------------------------- 5. frozen tables and networks
def packed_bytes(eng):
    torch.cuda.synchronize()
    out = []
    for net in (0, 1):
        d = eng.weights_debug(net)
        for name in ("x1", "x3", "bwd"):
            out.append(dev_tensor(getattr(d, name), (getattr(d, name + "_bytes") // 2,), "<i2").clone())
    return out


def test_frozen_tables_and_networks(env):
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    fit = fitter(env, fit=("latent",))
    p0, e0, l0 = fit.poses.clone(), fit.expressions.clone(), fit.latents.clone()
    models0 = [t.detach().clone() for m in (fit.mc, fit.mf) for t in m.parameters()]
    fit.step([0, 1], 64)
    packed0 = packed_bytes(eng)
    for i in range(10):
        fit.step([i % 6, (i + 2) % 6, 5], 64)
    torch.cuda.synchronize()
    assert torch.equal(fit.poses, p0) and torch.equal(fit.expressions, e0) and not torch.equal(fit.latents, l0)
    assert all(torch.equal(a, b.detach()) for a, b in zip(models0, [t for m in (fit.mc, fit.mf) for t in m.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(packed0, packed_bytes(eng)))
    for t in ("pose", "expression"):
        assert not fit._table(fit.exp_avg, t).any() and not fit._table(fit.grads, t).any()


def test_interleaved_trainer_step_does_not_change_the_fit(env):
    """A FusedTrainer step (which re-packs its own weights) between two fitting steps: the fitter re-packs its networks before
    its next step, eager or replayed, which then equals the step without the interleaving bit for bit."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    frs, images, poses, exprs, lats = frames(4, 32, seed=9)
    tr = fused_train.FusedTrainer(make_model(nerf, O.random_init_params(200), dev), make_model(nerf, O.random_init_params(201), dev),
                                  n_latent=4, num_coarse=64, num_fine=64, perturb=False, noise_std=0.0)
    data = ray_sampler.TrainImages(images.to(dev), poses, exprs, BOXES[:4], frs[0]["intrinsics"], background=frs[0]["bg"], device=dev)
    for graph in (False, True):
        runs = []
        for interleave in (False, True):
            fit = fitter(env, perturb=False, noise_std=0.0)
            if graph:
                fit.capture(2, 64, max_rounds=16, device_draws=False)
            step = (lambda d, f=fit: f.step_graph([1, 3], draws=d)) if graph else (lambda d, f=fit: f.step([1, 3], 64, draws=d, max_rounds=16))
            step(draws_for(dev, 2, 64, 16, 1))
            if interleave:
                tr.step_images(data, [0, 2], 64)
            loss = step(draws_for(dev, 2, 64, 16, 2)).clone()
            torch.cuda.synchronize()
            runs.append((loss, fit.params.clone(), fit.exp_avg_sq.clone()))
        assert all(torch.equal(a, b) for a, b in zip(*runs)), graph


# ----------------------------------------------------------------------------------------------------------------- 6. aliasing
def test_writes_into_the_tables_reach_the_next_step(env):
    nerf, _engine, fused_train, ray_sampler, dev = env
    fit = fitter(env, perturb=False, noise_std=0.0)
    t_new = torch.tensor([0.05, -0.1, 0.9], device=dev)
    fit.gradients([2, 1], 64, max_rounds=16)
    assert not torch.equal(fit._last["ray_origins"][:64], t_new.expand(64, 3))
    fit.poses[2, 3::4] = t_new
    fit.expressions[2] = 0.25
    fit.gradients([2, 1], 64, max_rounds=16)
    torch.cuda.synchronize()
    assert torch.equal(fit._last["ray_origins"][:64], t_new.expand(64, 3))
    assert (fit._last["expressions"][0] == 0.25).all()
    fit.capture(2, 64, max_rounds=16)
    fit.poses[1, 3::4] = -t_new
    fit.latents[1] = 0.5
    fit.step_graph([1, 2])
    torch.cuda.synchronize()
    sb = fit._graph["sb"]
    assert torch.equal(sb["ray_origins"][:64], (-t_new).expand(64, 3)) and (sb["latents"][0] == 0.5).all()


# ------------------------------------------------------------------------------------------------------------------ 7. capture
def test_replays_equal_eager_steps(env, monkeypatch):
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    fe, fg = fitter(env, perturb=False, noise_std=0.0), fitter(env, perturb=False, noise_std=0.0)
    fg.capture(3, 64, max_rounds=16, device_draws=False)
    for i in range(10):
        ids = [4, 1, 4] if i % 2 == 0 else [0, 5, 2]
        d = draws_for(dev, 3, 64, 16, 60 + i)
        la = fe.step(ids, 64, draws=d, max_rounds=16).clone()
        lb = (fg.step(ids, 64, draws=d, max_rounds=16) if i in (3, 7) else fg.step_graph(torch.tensor(ids, dtype=torch.int32, device=dev),
                                                                                          draws=d)).clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb), i
        for name in ("params", "grads", "exp_avg", "exp_avg_sq"):
            assert torch.equal(getattr(fe, name), getattr(fg, name)), (i, name)
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            f = fitter(env)
            torch.manual_seed(77)
            losses = [f.step([3, 1, 3], 64).clone() for _ in range(3)]
            torch.cuda.synchronize()
            runs.append((torch.stack(losses), f.params.clone()))
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_replay_after_reallocation_raises_and_short_selections(env):
    nerf, _engine, fused_train, ray_sampler, dev = env
    fit = fitter(env)
    fit.capture(2, 32)
    fit.step_graph([0, 1])
    big = fitter(env)
    big.step(list(range(6)) * 8, 256)  # more images and rays per step: the sampler and training buffers grow
    with pytest.raises(RuntimeError, match="capture again"):
        fit.step_graph([0, 1])
    # a 1x2-pixel box holding 90 % of the mass: one round cannot find 2048 distinct pixels
    nerf_, _e, _f, _r, _d = env
    frs, images, poses, exprs, lats = frames(2, 64)
    short = nerf.FusedFitter(fit.mc, fit.mf, images.to(dev), [(10, 11, 12, 14), (10, 50, 12, 44)], frs[0]["intrinsics"], poses, exprs, lats,
                             num_coarse=32, num_fine=32)
    p0 = short.params.clone()
    with pytest.raises(RuntimeError, match="fewer than"):
        short.step([0, 1], 2048, max_rounds=1)
    assert torch.equal(short.params, p0) and not short.grads.any() and short.iter == 0
    short.capture(2, 2048, has_background=False, max_rounds=1)
    loss = short.step_graph([0, 1])
    torch.cuda.synchronize()
    assert int(short.shortfall[0]) > 0 and torch.isfinite(loss).all() and torch.isfinite(short.params).all()


# ------------------------------------------------------------------------------------------------------------ 8. memory budget
def test_step_over_the_memory_budget(env, monkeypatch):
    nerf, _engine, fused_train, ray_sampler, dev = env
    res = []
    for budget in ("20000", "48"):
        monkeypatch.setenv("NFB_TRAIN_MEM_MB", budget)
        fit = fitter(env)
        torch.manual_seed(5)
        loss = fit.gradients([0, 2, 1, 2], 64, draws=draws_for(dev, 4, 64, 16, 3), max_rounds=16).clone()
        torch.cuda.synchronize()
        res.append((loss, [fit._table(fit.grads, t).clone() for t in ("pose", "expression", "latent")]))
    (l1, g1), (l2, g2) = res
    assert float((l1 - l2).abs().max()) < 1e-5
    for a, b in zip(g1, g2):
        assert float((a - b).abs().max()) <= 3e-3 * max(float(a.abs().max()), 1e-12)


# ------------------------------------------------------------------------------------------------------------- 9. launch count
COMBOS = [("pose",), ("expression",), ("latent",), ("pose", "expression"), ("pose", "latent"), ("expression", "latent"),
          ("pose", "expression", "latent")]


def test_launches_per_step_are_the_documented_ones(env):
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    doc = re.sub(r"\s+", " ", nerf.FusedFitter.step.__doc__)
    for combo in COMBOS:
        want = int(re.search(re.escape("(" + ", ".join(combo) + ")") + r": (\d+)", doc).group(1))
        fit = fitter(env, fit=combo)
        fit.step([0, 3, 0], 64)  # sizes the sampler's scratch
        l0 = eng.launch_count()
        fit.step([0, 3, 0], 64)
        got = eng.launch_count() - l0
        print(f"{combo}: {got} launches per step")
        assert got == want, (combo, got, want)
        fit.capture(3, 64)
        l0 = eng.launch_count()
        fit.step_graph([1, 2, 4])
        torch.cuda.synchronize()
        assert eng.launch_count() == l0
