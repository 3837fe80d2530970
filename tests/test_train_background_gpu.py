"""A learned background in the fused K-image training step (NFB_TRAIN_BACKGROUND): nfb_background_rows_grad and
nfb_loss_background_grad against their documented FP32 orders bit for bit and against float64, on real sampler batches
(repeats, incomplete selections, out-of-range slots, NaN gradients, data-parallel slices); one step against autograd +
torch.optim.Adam with the background as its own parameter group; the table read in place; graph replays against eager steps;
the launch counts; data-parallel ranks played by one process; reproducibility; and a trainer without a background unchanged."""
import re

import numpy as np
import pytest
import torch

import nerface_oracle as O
from test_train_background_cpu import background_rows_fp32, gamma, loss_background_fp32, pixel_keys
from test_train_images_gpu import dataset, make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train, ray_sampler
    return nerf, _engine, fused_train, ray_sampler, torch.device("cuda", 0)


def plain_dataset(ray_sampler, dev, n_images, H, W, bboxs, seed=0):
    """The training set without a background of its own (what a trainer that learns one takes), and the frames."""
    data, frs, images = dataset(ray_sampler, dev, n_images, H, W, bboxs, seed=seed)
    return ray_sampler.TrainImages(images.to(dev), data.poses, data.expressions, bboxs, frs[0]["intrinsics"], device=dev), frs, images


def sample_rc(eng, data, ids, n, draws, rounds, dev):
    """pixel_rc [K*n,2] (and the state) of one sampler call."""
    N = len(ids) * n
    out = dict(pixel_rc=torch.full((N, 2), -7, device=dev, dtype=torch.int32), state=torch.zeros(len(ids), 3, device=dev, dtype=torch.int32))
    eng.sample_images(data, torch.tensor(ids, dtype=torch.int32, device=dev), n, draws, rounds, torch.zeros(data.n_images, 32, device=dev), out)
    torch.cuda.synchronize()
    return out


def rows_on_device(eng, rc, H, W, gr, gl, dev, table0=None):
    t = torch.zeros(H, W, 3, device=dev) if table0 is None else table0.clone()
    eng.background_rows_grad(rc, H, W, gr, gl, t)
    torch.cuda.synchronize()
    return t.reshape(-1, 3).cpu().numpy()


def check_f64(got, rc, H, W, gr, gl):
    """Every row within gamma(2 m) * sum|g| of the float64 sum of its m rays (one rounding per g_r, one per add)."""
    key = pixel_keys(rc, H, W)
    g = gr.astype(np.float64) + (0.0 if gl is None else gl.astype(np.float64))
    fin = np.isfinite(g).all(1)
    order = np.argsort(key, kind="stable")
    ks, starts = np.unique(key[order], return_index=True)
    ends = list(starts[1:]) + [len(order)]
    hit = np.zeros(H * W, dtype=bool)
    for kk, a, b in zip(ks, starts, ends):
        if kk < 0:
            continue
        rays = order[a:b]
        hit[kk] = True
        if not fin[rays].all():
            continue
        want, mag = g[rays].sum(0), np.abs(g[rays]).sum(0)
        assert (np.abs(got[kk] - want) <= gamma(2 * len(rays)) * mag + 1e-45).all(), (kk, len(rays))
    assert not got[~hit].any()


@pytest.mark.parametrize("K,n", [(1, 1), (1, 2048), (2, 7), (8, 2048), (64, 7), (64, 2048)])
def test_rows_follow_the_documented_order(env, K, n):
    """Bit for bit background_rows_fp32 on sampler batches with repeated image indices (pixels collide across slots), with and
    without the loss term, NaN on one ray; within gamma(hits) of float64."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    H = W = 64
    bboxs = [(10, 50, 12, 44), (0, 64, 0, 64), (20, 40, 8, 60)]
    data, _, _ = plain_dataset(ray_sampler, dev, 3, H, W, bboxs)
    ids = [int(i) for i in np.random.default_rng(K + n).integers(0, 3, K)]
    g = torch.Generator(device=dev).manual_seed(K * 7 + n)
    draws = torch.rand(K * 16 * n, dtype=torch.float64, device=dev, generator=g)
    rc = sample_rc(eng, data, ids, n, draws, 16, dev)["pixel_rc"]
    rng = np.random.default_rng(n)
    scale = (10.0 ** rng.integers(-6, 1, (K * n, 1))).astype(np.float32)
    gr = (rng.standard_normal((K * n, 3)) * scale).astype(np.float32)
    gl = (rng.standard_normal((K * n, 3)) * scale * 0.01).astype(np.float32)
    gr[K * n // 2, 2] = np.nan
    rcn = rc.cpu().numpy()
    for gl_ in (None, gl):
        t0 = torch.randn(H, W, 3, device=dev) * 1e-3  # rows are ADDED to
        got = rows_on_device(eng, rc, H, W, torch.from_numpy(gr).to(dev), None if gl_ is None else torch.from_numpy(gl_).to(dev), dev, t0)
        want = background_rows_fp32(rcn, H, W, gr, gl_, t0.cpu().numpy())
        assert np.array_equal(got, want, equal_nan=True), (K, n)
        got0 = rows_on_device(eng, rc, H, W, torch.from_numpy(gr).to(dev), None if gl_ is None else torch.from_numpy(gl_).to(dev), dev)
        check_f64(got0, rcn, H, W, gr, gl_)
        nan_px = pixel_keys(rcn, H, W)[K * n // 2]
        assert np.isnan(got0[nan_px, 2]) and np.isfinite(np.delete(got0, nan_px, axis=0)).all()


def test_rows_at_incomplete_selections_out_of_range_slots_and_rank_slices(env):
    """A tiny box with max_rounds = 1 (slots j >= n_found repeat pixel j % n_found), an out-of-range image slot (pixel_rc -1: adds
    nothing), and slices of W = 2, 3, 4, 8 ranks that cut slots and repeat groups: every rank's rows bit for bit the restatement
    of its slice, and their rank-order sum within the float64 bound of the whole batch."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    H = W = 64
    bboxs = [(10, 14, 12, 15), (10, 50, 12, 44)]
    data, _, _ = plain_dataset(ray_sampler, dev, 2, H, W, bboxs)
    ids, n = [0, 1, 5, 0], 600
    draws = torch.rand(len(ids) * n, dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    out = sample_rc(eng, data, ids, n, draws, 1, dev)
    found = out["state"][:, 0].cpu().tolist()
    assert found[0] < n and found[3] < n  # incomplete: repeat groups
    rcn = out["pixel_rc"].cpu().numpy()
    assert (rcn[2 * n:3 * n] == -1).all()  # the out-of-range slot
    rng = np.random.default_rng(11)
    N = len(ids) * n
    gr = rng.standard_normal((N, 3)).astype(np.float32)
    gl = (rng.standard_normal((N, 3)) * 0.1).astype(np.float32)
    got = rows_on_device(eng, out["pixel_rc"], H, W, torch.from_numpy(gr).to(dev), torch.from_numpy(gl).to(dev), dev)
    assert np.array_equal(got, background_rows_fp32(rcn, H, W, gr, gl))
    check_f64(got, rcn, H, W, gr, gl)
    for world in (2, 3, 4, 8):
        per = N // world
        assert N % world == 0
        total = np.zeros((H * W, 3), dtype=np.float32)
        for r in range(world):
            sl = slice(r * per, (r + 1) * per)
            part = rows_on_device(eng, out["pixel_rc"][sl].contiguous(), H, W, torch.from_numpy(gr[sl]).to(dev),
                                  torch.from_numpy(gl[sl]).to(dev), dev)
            assert np.array_equal(part, background_rows_fp32(rcn[sl], H, W, gr[sl], gl[sl])), (world, r)
            total = (total + part).astype(np.float32)
        check_f64(total, rcn, H, W, gr, gl)


def test_loss_follows_its_order_and_shards_sum(env):
    """The loss and both gradients bit for bit loss_background_fp32; the loss within the gamma bound of float64; the shares of a
    sharded batch (n_total = the whole batch) sum to the batch loss within rounding, and their gradients are the batch's."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    rng = np.random.default_rng(5)
    for n in (1, 7, 2048, 5000):
        bg, t = rng.random((n, 3)).astype(np.float32), rng.random((n, 3)).astype(np.float32)
        w = rng.random(n).astype(np.float32)
        dv = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
        gb, gw, loss = torch.empty(n, 3, device=dev), torch.empty(n, device=dev), torch.full((1,), 0.25, device=dev)
        eng.loss_background_grad(dv(bg), dv(t), dv(w), n, 0.001, gb, gw, loss)
        torch.cuda.synchronize()
        wb, ww, wl = loss_background_fp32(bg, t, w, n, 0.001, 0.25)
        assert np.array_equal(gb.cpu().numpy(), wb) and np.array_equal(gw.cpu().numpy(), ww) and float(loss) == float(wl), n
        d = bg.astype(np.float64) - t.astype(np.float64)
        want = 0.001 / n * float((w * (d * d).sum(1)).sum())
        loss.zero_()
        eng.loss_background_grad(dv(bg), dv(t), dv(w), n, 0.001, gb, gw, loss)
        assert abs(float(loss) - want) <= gamma(n + 40) * want
        if n % 4 == 0:
            shares = torch.zeros(1, device=dev)
            for r in range(4):
                sl = slice(r * n // 4, (r + 1) * n // 4)
                gbs, gws = torch.empty(n // 4, 3, device=dev), torch.empty(n // 4, device=dev)
                eng.loss_background_grad(dv(bg[sl]), dv(t[sl]), dv(w[sl]), n, 0.001, gbs, gws, shares)
                assert torch.equal(gbs, gb[sl]) and torch.equal(gws, gw[sl])
            assert abs(float(shares) - want) <= gamma(n + 80) * want


def _cfg(nerf, num_fine):
    blk = dict(num_coarse=64, num_fine=num_fine, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=65536)
    return nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))


def _learner(nerf, fused_train, dev, n_latent, lat0, bg0, weight, num_fine, precision=None, noisy=True):
    mf = make_model(nerf, O.random_init_params(101), dev) if num_fine > 0 else None
    return fused_train.FusedTrainer(make_model(nerf, O.random_init_params(100), dev), mf, n_latent=n_latent, lr=5e-4,
                                    lr_decay_steps=250.0, lr_decay_factor=0.1, num_coarse=64, num_fine=num_fine, perturb=noisy,
                                    noise_std=0.1 if noisy else 0.0, latent_reg=0.005, latent_codes=lat0, precision=precision, background=bg0,
                                    background_loss=weight)


def _ulp_close(a, b, tol):
    a, b = a.double(), b.double()
    ulp = torch.from_numpy(np.spacing(np.abs(b.cpu().numpy()).astype(np.float32)).astype(np.float64)).to(a.device)
    return bool(((a - b).abs() <= tol + ulp).all())


@pytest.mark.parametrize("ids,precision,weight,num_fine", [
    ([1], "fast", 0.001, 64), ([2], "exact_grad", 0.0, 0), ([0, 0], "exact", 0.001, 64), ([2, 0], "fast", 0.0, 0),
    ([0, 1, 2, 0, 1, 0, 2, 2], "exact_grad", 0.001, 64), ([1, 1, 0, 2, 0, 1, 2, 1], "fast", 0.001, 0)])
def test_step_matches_autograd_and_torch_adam(env, ids, precision, weight, num_fine, monkeypatch):
    """One step's gradients against autograd through the background gathered at the trainer's own pixels (bitwise where a pixel
    is hit once, within gamma(hits) otherwise; parameters and latents within 1e-6 of each tensor's max), then Adam against
    torch.optim.Adam with groups [params + latents, bg]: tables within 7.5e-9 + 1 ulp after one step, losses within 2e-6 over 10
    steps (K = 1 uses run_one_iter_of_nerf, K >= 2 render_frames)."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    from nerf._engine import PARAM_ORDER
    H = W = 32
    bboxs = [(8, 24, 6, 26), (4, 20, 10, 30), (0, 32, 0, 32)]
    data, frs, images = plain_dataset(ray_sampler, dev, 3, H, W, bboxs)
    # a handle of its own: after an exact-grad forward every re-pack of a handle takes one more launch, which other tests count
    eng = _engine.Renderer(dev)
    monkeypatch.setitem(_engine._renderers, ("cuda", dev.index), eng)
    k, n, rounds, steps = len(ids), 64, 16, 10
    lr0, decay, factor, reg = 5e-4, 250.0, 0.1, 0.005
    lat0 = torch.randn(3, 32, generator=torch.Generator().manual_seed(2)) * 0.1
    bg0 = images.mean(0)  # the reference's initialisation
    g = torch.Generator(device=dev).manual_seed(8)
    draws = [torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=g) for _ in range(steps)]
    cfg = _cfg(nerf, num_fine)
    old = nerf.get_precision()
    nerf.set_precision(precision)
    try:
        # ---- autograd + torch.optim.Adam, the background its own parameter group
        mc = make_model(nerf, O.random_init_params(100), dev)
        mf = make_model(nerf, O.random_init_params(101), dev) if num_fine > 0 else None
        nets = list(mc.parameters()) + (list(mf.parameters()) if mf is not None else [])
        latent_codes = lat0.clone().to(dev).requires_grad_(True)
        bg = bg0.clone().to(dev).requires_grad_(True)
        opt = torch.optim.Adam([{"params": nets + [latent_codes]}, {"params": [bg], "lr": lr0}], lr=lr0)
        ids_t = torch.tensor(ids, device=dev)
        ref_losses, rcs = [], []
        for i in range(steps):
            b = sample_rc(eng, data, ids, n, draws[i], rounds, dev)
            rc = b["pixel_rc"].long()
            rcs.append(b["pixel_rc"])
            tgt = images.to(dev)[ids_t.repeat_interleave(n), rc[:, 0], rc[:, 1]]
            bgr = bg[rc[:, 0], rc[:, 1]]
            intr = frs[0]["intrinsics"]
            torch.manual_seed(700 + i)
            sb = _sample_rays(eng, data, ids, n, draws[i], rounds, dev)
            if k == 1:
                out = nerf.run_one_iter_of_nerf(H, W, intr, mc, mf, sb["ray_origins"], sb["ray_directions"], cfg, mode="train",
                                                expressions=data.expressions[ids[0]], background_prior=bgr,
                                                latent_code=latent_codes[ids[0]])
            else:
                out = nerf.render_frames(sb["ray_origins"], sb["ray_directions"], sb["frame_index"], data.expressions[ids_t],
                                         latent_codes[ids_t], mc, mf, cfg, mode="train", background_prior=bgr)
            coarse = torch.nn.functional.mse_loss(out[0], tgt)
            fine = torch.nn.functional.mse_loss(out[3], tgt) if num_fine > 0 else torch.zeros((), device=dev)
            loss = coarse + fine + (reg / k) * sum(torch.norm(latent_codes[j]) for j in ids)
            if weight > 0:
                e = torch.nn.functional.mse_loss(bgr, tgt, reduction="none").sum(1)
                loss = loss + torch.mean(e * out[6]) * weight
            loss.backward()
            if i == 0:
                ref_grads = [[(dict(m.named_parameters())[q].grad.clone() if dict(m.named_parameters())[q].grad is not None else None)
                              for q in PARAM_ORDER] for m in ([mc] + ([mf] if mf is not None else []))]
                ref_lat, ref_bg = latent_codes.grad.clone(), bg.grad.clone()
            opt.step()
            opt.zero_grad()
            for gp in opt.param_groups:
                gp["lr"] = lr0 * factor ** (i / decay)
            if i == 0:
                ref_p1 = dict(lat=latent_codes.detach().clone(), bg=bg.detach().clone())
            ref_losses.append((float(coarse.detach()), float(fine.detach())))

        # ---- the fused step: gradients of step 0 first
        tr = _learner(nerf, fused_train, dev, 3, lat0, bg0, weight, num_fine)
        tr._own_engine()
        dv = tr._images_data(data)
        sbf = tr._images_buffers(dv, k, n)
        sbf["img"].copy_(ids_t)
        tr._images_sample(dv, sbf, n, draws[0], rounds)
        torch.manual_seed(700)
        tr._images_gradients(sbf, k, n)
        torch.cuda.synchronize()
        assert torch.equal(sbf["pixel_rc"], rcs[0])
        rc0 = rcs[0].long()
        assert torch.equal(sbf["background"], bg0.to(dev)[rc0[:, 0], rc0[:, 1]])  # read in place from the bucket's rows
        for gs_ref, gs in zip(ref_grads, (tr._gc, tr._gf)):
            for name, a, b_ in zip(PARAM_ORDER, gs_ref, gs):
                if a is not None and b_ is not None:
                    assert float((a - b_).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-12), name
        if k >= 2:
            gtab = tr._latent_grads()
            assert float((ref_lat - gtab).abs().max()) <= 1e-6 * float(ref_lat.abs().max())
        key = torch.from_numpy(pixel_keys(rcs[0].cpu().numpy(), H, W))
        hits = torch.bincount(key[key >= 0], minlength=H * W).to(dev)
        got_bg, want_bg = tr._bg_grads.reshape(-1, 3), ref_bg.reshape(-1, 3)
        once = hits == 1
        assert torch.equal(got_bg[once], want_bg[once]), precision
        assert not got_bg[hits == 0].any()
        rep = hits > 1
        if bool(rep.any()):
            # both sides sum the same per-ray terms in an order of their own: within 2 gamma(hits) * sum|terms| <= ... |row|
            mag = torch.zeros_like(got_bg)
            g_ray = tr.grads.new_zeros(k * n, 3)
            g_ray.copy_(sbf["g_bg"] + (sbf["g_bgl"] if weight > 0 else 0.0))
            mag.index_add_(0, key.to(dev).clamp(min=0), g_ray.abs())
            m = hits.double()[:, None]
            bound = 2 * m * 2.0 ** -24 / (1 - 2 * m * 2.0 ** -24) * mag.double()
            assert bool(((got_bg.double() - want_bg.double()).abs() <= bound)[rep].all())
        tr.grads.zero_()

        # ---- ten steps: one against torch.optim.Adam, then the loss curves
        fused = []
        for i in range(steps):
            torch.manual_seed(700 + i)
            lv = tr.step_images(data, ids, n, draws=draws[i], max_rounds=rounds)
            fused.append(tuple(float(v) for v in lv))
            if i == 0:
                assert _ulp_close(tr.background, ref_p1["bg"], 7.5e-9)
                assert _ulp_close(tr.latent_codes, ref_p1["lat"], 7.5e-9)
        for (a, c_), (b_, d) in zip(ref_losses, fused):
            assert abs(a - b_) < 2e-6 and abs(c_ - d) < 2e-6, (a, b_, c_, d)
    finally:
        nerf.set_precision(old)


def _sample_rays(eng, data, ids, n, draws, rounds, dev):
    N = len(ids) * n
    z = lambda *s, dt=torch.float32: torch.zeros(s, device=dev, dtype=dt)  # noqa: E731
    out = dict(ray_origins=z(N, 3), ray_directions=z(N, 3), frame_index=z(N, dt=torch.int32))
    eng.sample_images(data, torch.tensor(ids, dtype=torch.int32, device=dev), n, draws, rounds, torch.zeros(data.n_images, 32, device=dev), out)
    return out


def test_table_is_read_in_place_eager_and_replayed(env, monkeypatch):
    """A step's background rays are trainer.background at the sampled pixels, bit for bit; a write into trainer.background
    between steps changes the next step's rays, eager and replayed; the caller's TrainImages keeps no background."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    data, frs, images = plain_dataset(ray_sampler, dev, 3, 32, 32, [(8, 24, 6, 26)] * 3)
    lat0 = torch.zeros(3, 32)
    for k in (1, 4):
        ids = [0, 2, 1, 2][:k]
        te = _learner(nerf, fused_train, dev, 3, lat0, images.mean(0), 0.001, 64)
        tg = _learner(nerf, fused_train, dev, 3, lat0, images.mean(0), 0.001, 64)
        tg.capture_images(data, k, 64, max_rounds=16, device_draws=False)
        assert data.background is None and data.desc.background is None
        g = torch.Generator(device=dev).manual_seed(k)
        for i in range(3):
            draws = torch.rand(k * 16 * 64, dtype=torch.float64, device=dev, generator=g)
            for t in (te, tg):
                t.background[:, :, 1] = 0.25 * (i + 1)  # a write between steps
            before = {id(t): t.background.clone() for t in (te, tg)}
            te.step_images(data, ids, 64, draws=draws, max_rounds=16)
            tg.step_images_graph(ids, draws=draws)
            torch.cuda.synchronize()
            for t, sb in ((te, te._image_bufs[(k, 64, True)]), (tg, tg._igraph["sb"])):
                rc = sb["pixel_rc"].long()
                assert torch.equal(sb["background"], before[id(t)][rc[:, 0], rc[:, 1]]), (k, i)
                assert (sb["background"][:, 1] == 0.25 * (i + 1)).all()


def test_graph_replays_equal_eager_steps_and_launch_counts(env, monkeypatch):
    """10 replays equal 10 eager steps bit for bit (bucket, moments, losses, loss[2]); nfb_launch_count per eager step is the
    documented count (18 / 21 learned, 19 / 22 supervised); a replay issues no launch from the host; without background= the
    bucket and the counts are today's (16 / 19)."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    eng = _engine.Renderer(dev)  # a handle of its own: one that ran an exact-grad forward takes one more launch per re-pack
    monkeypatch.setitem(_engine._renderers, ("cuda", dev.index), eng)
    doc = fused_train.FusedTrainer.step_images.__doc__
    assert re.search(r"18 launches at K = 1 and 21 at K >= 2", doc) and "(+1: 19 and 22)" in doc
    data, frs, images = plain_dataset(ray_sampler, dev, 4, 32, 32, [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20), (0, 32, 0, 32)])
    lat0 = torch.randn(4, 32) * 0.1
    for weight in (0.0, 0.001):
        # without noise: an eager step draws it from torch's generator, a replay from the graph's Philox state
        te = _learner(nerf, fused_train, dev, 4, lat0, images.mean(0), weight, 64, noisy=False)
        tg = _learner(nerf, fused_train, dev, 4, lat0, images.mean(0), weight, 64, noisy=False)
        tg.capture_images(data, 4, 64, max_rounds=16, device_draws=False)
        g = torch.Generator(device=dev).manual_seed(13)
        for i in range(10):
            draws = torch.rand(4 * 16 * 64, dtype=torch.float64, device=dev, generator=g)
            step_ids = [3, 1, 3, 0] if i % 2 == 0 else [2, 2, 1, 0]
            la = te.step_images(data, step_ids, 64, draws=draws, max_rounds=16).clone()
            lb = tg.step_images_graph(torch.tensor(step_ids, dtype=torch.int32, device=dev), draws=draws).clone()
            torch.cuda.synchronize()
            assert torch.equal(la, lb) and torch.equal(te.loss, tg.loss), (weight, i)
            for name in ("params", "exp_avg", "exp_avg_sq"):
                assert torch.equal(getattr(te, name), getattr(tg, name)), (weight, i, name)
        assert (float(te.loss[2]) > 0.0) == (weight > 0.0)
        for ids, want in (([1], 18), ([0, 2], 21), ([0, 1, 2, 1], 21)):
            want += 1 if weight > 0 else 0
            te.step_images(data, ids, 64)
            l0 = eng.launch_count()
            te.step_images(data, ids, 64)
            assert eng.launch_count() - l0 == want, (weight, ids)
        tg.step_images_graph([1, 2, 0, 3], draws=torch.rand(4 * 16 * 64, dtype=torch.float64, device=dev))  # re-packs: te ran last
        l0 = eng.launch_count()
        tg.step_images_graph([1, 2, 0, 3], draws=torch.rand(4 * 16 * 64, dtype=torch.float64, device=dev))
        torch.cuda.synchronize()
        assert eng.launch_count() == l0
    plain = fused_train.FusedTrainer(make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev),
                                      n_latent=4)
    learned = _learner(nerf, fused_train, dev, 4, None, images.mean(0), 0.0, 64)
    assert plain.params.numel() == plain.lat_off + 4 * 32 and plain.background is None
    assert learned.bg_off == (plain.params.numel() + 255) // 256 * 256 and learned.lat_off == plain.lat_off
    assert learned.params.numel() == learned.bg_off + 32 * 32 * 3
    withbg, _, _ = dataset(ray_sampler, dev, 4, 32, 32, [(8, 24, 6, 26)] * 4)
    for ids, want in (([1], 16), ([0, 2], 19)):
        plain.step_images(withbg, ids, 64)
        l0 = eng.launch_count()
        plain.step_images(withbg, ids, 64)
        assert eng.launch_count() - l0 == want


@pytest.mark.parametrize("world", [2, 4, 8])
def test_data_parallel_ranks_on_one_gpu(env, world, monkeypatch):
    """One process plays `world` ranks (explicit rank=, the collective a rank-order sum of the buckets): every rank's batch is
    bitwise the single process's, the summed background rows lie within the float64 bound of the per-ray terms, and every rank
    holds the same bucket before Adam."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    data, frs, images = plain_dataset(ray_sampler, dev, 3, 32, 32, [(8, 24, 6, 26), (4, 20, 10, 30), (0, 32, 0, 32)])
    ids, n, rounds = [0, 2, 0, 1], 64, 16
    k, N = len(ids), len(ids) * n
    lat0 = torch.randn(3, 32) * 0.1
    draws = torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    one = _learner(nerf, fused_train, dev, 3, lat0, images.mean(0), 0.001, 64)
    one._own_engine()
    d1 = one._images_data(data)
    sb1 = one._images_buffers(d1, k, n)
    sb1["img"].copy_(torch.tensor(ids, dtype=torch.int32))
    one._images_sample(d1, sb1, n, draws, rounds)
    torch.manual_seed(5)
    one._images_gradients(sb1, k, n)
    torch.cuda.synchronize()
    ranks, buckets, rays = [], [], []
    for r in range(world):
        t = _learner(nerf, fused_train, dev, 3, lat0, images.mean(0), 0.001, 64)
        t._own_engine()
        dr = t._images_data(data)
        sb = t._images_buffers(dr, k, n)
        sb["img"].copy_(torch.tensor(ids, dtype=torch.int32))
        t._images_sample(dr, sb, n, draws, rounds)
        torch.manual_seed(5)
        t._images_gradients(sb, k, n, world, r)
        torch.cuda.synchronize()
        for name in ("pixel_rc", "ray_origins", "ray_directions", "target", "background", "frame_index"):
            assert torch.equal(sb[name], sb1[name]), (r, name)
        ranks.append((t, sb))
        buckets.append(t.grads.clone())
        rays.append((sb["g_bg"] + sb["g_bgl"]).clone())
    total = buckets[0].clone()
    for b in buckets[1:]:
        total += b
    for t, sb in ranks:  # the collective (a rank-order sum), then the regulariser: every rank holds the same bucket before Adam
        t.grads.copy_(total)
        t._images_regulariser(sb, k)
    torch.cuda.synchronize()
    assert all(torch.equal(t.grads, ranks[0][0].grads) for t, _ in ranks)
    per = N // world
    g_ray = torch.cat([rays[r][r * per:(r + 1) * per] for r in range(world)]).cpu().numpy()
    bg_rows = total[one.bg_off:].reshape(-1, 3).cpu().numpy()
    rcn = sb1["pixel_rc"].cpu().numpy()
    check_f64(bg_rows, rcn, 32, 32, g_ray.astype(np.float32), None)
    whole = one.grads[one.bg_off:].reshape(-1, 3).cpu().numpy()
    assert np.array_equal(whole, background_rows_fp32(rcn, 32, 32, one._image_bufs[(k, n, True)]["g_bg"].cpu().numpy(),
                                                      one._image_bufs[(k, n, True)]["g_bgl"].cpu().numpy()))


def test_seeded_runs_repeat_under_deterministic_algorithms(env, monkeypatch):
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    data, frs, images = plain_dataset(ray_sampler, dev, 3, 32, 32, [(8, 24, 6, 26)] * 3)
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            t = _learner(nerf, fused_train, dev, 3, torch.zeros(3, 32), images.mean(0), 0.001, 64)
            torch.manual_seed(77)
            losses = [t.step_images(data, [0, 2, 2], 64).clone() for _ in range(3)]
            torch.cuda.synchronize()
            runs.append((torch.stack(losses), t.loss.clone(), t.params.clone(), t.exp_avg_sq.clone()))
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(*runs):
        assert torch.equal(a, b)
