"""Training steps over rays of several images (NFB_TRAIN_IMAGES): the batched device sampler against nfb_sample_rays and numpy's
choice image by image, the K = 1 step against FusedTrainer.step / step_graph bit for bit, K >= 2 against nerf.render_frames +
torch MSE + the regulariser + torch.optim.Adam, the latent-table rows against their documented FP32 order and float64, the
captured step against the eager one, the launch count, and the step over the memory budget."""
import re

import numpy as np
import pytest
import torch

import nerface_oracle as O
from test_post_gpu import numpy_choice_with_recorded_draws

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train, ray_sampler
    return nerf, _engine, fused_train, ray_sampler, torch.device("cuda", 0)


def make_model(nerf, params, dev):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params)
    return m.to(dev)


def dataset(ray_sampler, dev, n_images, H, W, bboxs, host=False, seed=0):
    frs = [O.synthetic_frame(seed + i, H, W) for i in range(n_images)]
    g = torch.Generator().manual_seed(seed + 100)
    images = torch.rand(n_images, H, W, 3, generator=g)
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs])
    data = ray_sampler.TrainImages(images if host else images.to(dev), poses, exprs, bboxs, frs[0]["intrinsics"],
                                   background=frs[0]["bg"], device=dev)
    return data, frs, images


def batch_buffers(dev, k, n):
    N = k * n
    z = lambda *s, dt=torch.float32: torch.full(s, -7, device=dev, dtype=dt)  # noqa: E731  (not zero: unwritten slots show)
    return dict(img=None, ray_origins=z(N, 3), ray_directions=z(N, 3), target=z(N, 3), background=z(N, 3), pixel_rc=z(N, 2, dt=torch.int32),
                indices=z(N, dt=torch.int64), frame_index=z(N, dt=torch.int32), expressions=z(k, 76), latents=z(k, 32),
                state=z(k, 3, dt=torch.int32), shortfall=torch.zeros(k, device=dev, dtype=torch.int64))


def sample(eng, data, ids, n, draws, rounds, table, dev):
    out = batch_buffers(dev, len(ids), n)
    img = torch.tensor(ids, dtype=torch.int32, device=dev)
    eng.sample_images(data, img, n, draws, rounds, table, out)
    torch.cuda.synchronize()
    return out


def recorded_draws(data_flat_maps, ids, n, rounds, seed):
    """Per image: numpy's choice indices and the uniform draws it consumed, laid out as slice k of [K][rounds * n]."""
    buf = np.full((len(ids), rounds * n), 0.5)
    expected = []
    for k, i in enumerate(ids):
        exp, draws = numpy_choice_with_recorded_draws(data_flat_maps[i].size, n, data_flat_maps[i], seed + k)
        d = np.concatenate(draws)
        assert d.size <= rounds * n
        buf[k, :d.size] = d
        expected.append(exp)
    return buf, expected


@pytest.mark.parametrize("H,ids,bboxs,n,rounds", [
    (64, [0, 1, 1, 2], [(10, 50, 12, 44), (10, 14, 12, 15), (0, 64, 0, 64)], 2048, 64),  # box 1 needs many rounds
    (64, [2], [(10, 50, 12, 44), (20, 40, 8, 60), (5, 30, 30, 60)], 777, 8),
    (512, [3, 0, 2, 1, 0, 3, 2, 1], [(150, 400, 128, 380), (40, 300, 60, 500), (0, 512, 0, 512), (200, 260, 10, 400)], 2048, 16)])
def test_batched_sampler_equals_the_single_image_sampler(env, H, ids, bboxs, n, rounds):
    """Block k = nfb_sample_rays on image ids[k] fed draw slice k: indices (= numpy's choice), pixel_rc, rays, target and
    background bit for bit; frame index k on its rays; the conditioning rows are the tables' rows.  Pinned host images give the
    device images' targets."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    data, frs, images = dataset(ray_sampler, dev, len(bboxs), H, H, bboxs)
    host, _, _ = dataset(ray_sampler, dev, len(bboxs), H, H, bboxs, host=True)
    assert host.images.is_pinned() and not host.images.is_cuda
    flat = [ray_sampler.importance_map(H, H, bb, 0.9)[1] for bb in bboxs]
    k = len(ids)
    buf, expected = recorded_draws(flat, ids, n, rounds, seed=5)
    draws = torch.from_numpy(buf).to(dev)
    table = torch.randn(len(bboxs), 32, device=dev)
    out = sample(eng, data, ids, n, draws, rounds, table, dev)
    out_h = sample(eng, host, ids, n, draws, rounds, table, dev)
    st = out["state"].cpu()
    assert (st[:, 0] == n).all() and int(out["shortfall"].sum()) == 0
    single = ray_sampler.RaySampler(H, H, bboxs, size=n, device=dev)
    for j, i in enumerate(ids):
        s = slice(j * n, (j + 1) * n)
        ref = single.sample(i, draws=draws[j].contiguous(), pose=frs[i]["pose"], intrinsics=frs[i]["intrinsics"], image=images[i],
                            background=frs[0]["bg"], max_rounds=rounds)
        torch.cuda.synchronize()
        assert st[j].tolist() == ref["state"].cpu().tolist()
        assert np.array_equal(out["indices"][s].cpu().numpy(), expected[j])
        assert torch.equal(out["indices"][s], ref["indices"])
        assert torch.equal(out["pixel_rc"][s], ref["pixel_rc"])
        for name in ("ray_origins", "ray_directions", "target", "background"):
            assert torch.equal(out[name][s], ref[name]), (j, name)
            assert torch.equal(out_h[name][s], out[name][s]), (j, name)
        assert (out["frame_index"][s] == j).all()
        assert torch.equal(out["expressions"][j], data.expressions[i]) and torch.equal(out["latents"][j], table[i])


def test_short_selection_fills_counts_and_raises(env):
    """One round of draws cannot find 2048 distinct pixels when a 12-pixel box holds 90 % of the mass: the missing slots
    repeat the first selected pixels (finite batch), the shortfall counter says how many, and the eager step raises."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    bboxs = [(10, 14, 12, 15), (10, 50, 12, 44)]
    data, frs, images = dataset(ray_sampler, dev, 2, 64, 64, bboxs)
    n = 2048
    draws = torch.rand(2 * n, dtype=torch.float64, device=dev)
    out = sample(eng, data, [0, 1], n, draws, 1, torch.zeros(2, 32, device=dev), dev)
    found = out["state"][:, 0].cpu().tolist()
    assert found[0] < n and int(out["shortfall"][0]) == n - found[0] and int(out["shortfall"][1]) == n - found[1]
    for name in ("ray_origins", "ray_directions", "target", "background"):
        assert torch.isfinite(out[name]).all(), name
    idx = out["indices"][:n]
    j = torch.arange(found[0], n, device=dev)
    assert torch.equal(idx[found[0]:], idx[j % found[0]])
    tr = fused_train.FusedTrainer(make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev),
                                  n_latent=2, num_coarse=32, num_fine=32)
    with pytest.raises(RuntimeError, match="fewer than"):
        tr.step_images(data, [0, 1], n, max_rounds=1)
    assert float(tr.grads.abs().max()) == 0.0 and tr.iter == 0
    tr.capture_images(data, 2, n, max_rounds=1)
    loss = tr.step_images_graph([0, 1])
    torch.cuda.synchronize()
    assert int(tr.shortfall.sum()) > 0 and torch.isfinite(loss).all()


def _trainer(nerf, fused_train, dev, n_latent, noisy, latents=None):
    return fused_train.FusedTrainer(make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev),
                                    n_latent=n_latent, lr=5e-4, lr_decay_steps=250.0, lr_decay_factor=0.1, num_coarse=64, num_fine=64,
                                    perturb=noisy, noise_std=0.1 if noisy else 0.0, latent_reg=0.005, latent_codes=latents)


def test_one_image_step_is_the_existing_step(env):
    """K = 1 runs the single-frame kernels: step_images equals step() fed the sampled rays, and its graph equals step_graph(),
    bit for bit — loss, bucket, Adam moments — over 10 steps."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    bboxs = [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20)]
    data, frs, images = dataset(ray_sampler, dev, 3, 32, 32, bboxs)
    n, rounds = 64, 8
    lat0 = torch.randn(3, 32) * 0.1
    single = ray_sampler.RaySampler(32, 32, bboxs, size=n, device=dev)
    g = torch.Generator(device=dev).manual_seed(4)
    for noisy in (True, False):
        ta, tb = _trainer(nerf, fused_train, dev, 3, noisy, lat0), _trainer(nerf, fused_train, dev, 3, noisy, lat0)
        if not noisy:
            ta.capture(n)
            tb.capture_images(data, 1, n, max_rounds=rounds, device_draws=False)
        for i in range(10):
            img = (i * 2) % 3
            draws = torch.rand(rounds * n, dtype=torch.float64, device=dev, generator=g)
            b = single.sample(img, draws=draws, pose=frs[img]["pose"], intrinsics=frs[img]["intrinsics"], image=images[img],
                              background=frs[0]["bg"], max_rounds=rounds)
            args = (b["ray_origins"], b["ray_directions"], b["target"], data.expressions[img], img)
            torch.manual_seed(300 + i)
            la = (ta.step(*args, background=b["background"]) if noisy else ta.step_graph(*args, background=b["background"])).clone()
            torch.manual_seed(300 + i)
            lb = (tb.step_images(data, [img], n, draws=draws, max_rounds=rounds) if noisy else tb.step_images_graph([img], draws=draws)).clone()
            torch.cuda.synchronize()
            assert torch.equal(la, lb), (noisy, i, la, lb)
            for name in ("params", "grads", "exp_avg", "exp_avg_sq"):
                assert torch.equal(getattr(ta, name), getattr(tb, name)), (noisy, i, name)
        assert ta.iter == tb.iter == 10


@pytest.mark.parametrize("ids", [[0, 1], [2, 0, 2, 1], [0, 1, 2, 3, 4, 5, 1, 3]])
def test_multi_image_step_matches_the_reference_style_step(env, ids):
    """K >= 2 against nerf.render_frames + torch MSE + (0.005 / K) * sum_k ||latent[ids[k]]|| + torch.optim.Adam on the same
    rays and noise: gradients within 1e-6 of each tensor's max, parameters within 1e-6 after one step, loss curves within 2e-6
    over 10 steps (the tolerances of test_fused_train_gpu.py's single-image comparison)."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    from nerf._engine import PARAM_ORDER
    bboxs = [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20), (0, 32, 0, 32), (12, 20, 12, 20), (2, 28, 4, 16)]
    data, frs, images = dataset(ray_sampler, dev, 6, 32, 32, bboxs)
    eng = _engine.renderer_for(dev)
    k, n, rounds, steps = len(ids), 64, 16, 10
    lr0, decay, factor, reg = 5e-4, 250.0, 0.1, 0.005
    lat0 = torch.randn(6, 32) * 0.1
    lat0[4] = 0.0  # a row at 0: its regulariser term is 0 (torch.norm's subgradient)
    g = torch.Generator(device=dev).manual_seed(8)
    draws = [torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=g) for _ in range(steps)]
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False, chunksize=65536)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))

    # ---- reference-style loop
    mc, mf = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
    latent_codes = lat0.clone().to(dev).requires_grad_(True)
    opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()) + [latent_codes], lr=lr0)
    ids_t = torch.tensor(ids, device=dev)
    ref_losses = []
    for i in range(steps):
        b = sample(eng, data, ids, n, draws[i], rounds, latent_codes.detach(), dev)
        torch.manual_seed(700 + i)
        out = nerf.render_frames(b["ray_origins"], b["ray_directions"], b["frame_index"], data.expressions[ids_t], latent_codes[ids_t],
                                 mc, mf, cfg, mode="train", background_prior=b["background"])
        coarse = torch.nn.functional.mse_loss(out[0], b["target"])
        fine = torch.nn.functional.mse_loss(out[3], b["target"])
        loss = coarse + fine + (reg / k) * sum(torch.norm(latent_codes[j]) for j in ids)
        loss.backward()
        if i == 0:
            ref_grads = [[dict(m.named_parameters())[q].grad for q in PARAM_ORDER] for m in (mc, mf)]
            ref_grads = [[t.clone() if t is not None else None for t in ts] for ts in ref_grads] + [latent_codes.grad.clone()]
        opt.step()
        opt.zero_grad()
        for gp in opt.param_groups:
            gp["lr"] = lr0 * factor ** (i / decay)
        if i == 0:
            ref_params1 = [p.detach().clone() for p in list(mc.parameters()) + list(mf.parameters())] + [latent_codes.detach().clone()]
        ref_losses.append((float(coarse), float(fine)))

    # ---- the fused K-image step
    tr = _trainer(nerf, fused_train, dev, 6, True, lat0)
    tr._own_engine()
    sb = tr._images_buffers(data, k, n)
    sb["img"].copy_(ids_t)
    tr._images_sample(data, sb, n, draws[0], rounds)
    torch.manual_seed(700)
    tr._images_gradients(sb, k, n)
    torch.cuda.synchronize()
    for gs_ref, gs in zip(ref_grads[:2], (tr._gc, tr._gf)):
        for name, a, b in zip(PARAM_ORDER, gs_ref, gs):
            assert (a is None) == (b is None), name
            if a is not None:
                assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-12), name
    gtab = tr.grads[tr.lat_off:].view(-1, 32)
    assert float((ref_grads[2] - gtab).abs().max()) <= 1e-6 * float(ref_grads[2].abs().max())
    assert all(float(gtab[j].abs().max()) == 0.0 for j in range(6) if j not in ids)
    tr.grads.zero_()
    fused = []
    for i in range(steps):
        torch.manual_seed(700 + i)
        lv = tr.step_images(data, ids, n, draws=draws[i], max_rounds=rounds)
        fused.append(tuple(float(v) for v in lv))
        if i == 0:
            worst = max(float((p - q.detach()).abs().max()) for p, q in zip(
                ref_params1, list(tr.mc.parameters()) + list(tr.mf.parameters()) + [tr.latent_codes]))
            print(f"K = {k}: fused vs render_frames + torch.optim.Adam after one step: max|d param| = {worst:.3e}")
            assert worst <= 1e-6
    for (a, b), (c, d) in zip(ref_losses, fused):
        assert abs(a - c) < 2e-6 and abs(b - d) < 2e-6, (a, c, b, d)


def latent_rows_fp32(glat, img, table, g0, w):
    """The documented order of nfb_latent_rows_grad in FP32 on the host (every op rounds once, as the kernel's)."""
    G = g0.clone()
    for k, r in enumerate(img):
        if 0 <= r < G.shape[0]:
            G[r] = G[r] + glat[k]
    lane = torch.arange(32)
    for k, r in enumerate(img):
        if not 0 <= r < G.shape[0] or w == 0.0:
            continue
        l = table[r]
        s = l * l
        for o in (16, 8, 4, 2, 1):
            s = s + s[lane ^ o]
        if float(s[0]) == 0.0:
            continue
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(s[0])
        G[r] = G[r] + (torch.tensor(w, dtype=torch.float32) * inv) * l
    return G


def test_latent_rows_follow_the_documented_order(env):
    """Bit for bit the documented FP32 order; within gamma(m) * sum|terms| of float64; rows not named exactly 0; a zero latent
    adds no term; an out-of-range index adds nothing."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    g = torch.Generator().manual_seed(21)
    rows = 10
    table = torch.randn(rows, 32, generator=g) * 0.3
    table[3] = 0.0
    for img in ([1], [2, 2, 5, 3, 7, 2], [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 3, 3, 12, -1] + list(range(50))[:40]):
        k = len(img)
        glat = torch.randn(k, 32, generator=g) * 10.0 ** torch.randint(-6, 1, (k, 1), generator=g).float()
        w = 0.005 / k
        got = torch.zeros(rows, 32, device=dev)
        eng.latent_rows_grad(glat.to(dev), torch.tensor(img, dtype=torch.int32, device=dev), table.to(dev), got, w)
        torch.cuda.synchronize()
        got = got.cpu()
        want = latent_rows_fp32(glat, img, table, torch.zeros(rows, 32), w)
        assert torch.equal(got, want), img
        ref, mag = torch.zeros(rows, 32, dtype=torch.float64), torch.zeros(rows, 32, dtype=torch.float64)
        t64 = table.double()
        for j, r in enumerate(img):
            if 0 <= r < rows:
                ref[r] += glat[j].double()
                mag[r] += glat[j].double().abs()
                nrm = float(t64[r].norm())
                if nrm > 0:
                    ref[r] += w * t64[r] / nrm
                    mag[r] += (w * t64[r] / nrm).abs()
        m = 2 * k + 40
        gam = m * 2.0 ** -24 / (1 - m * 2.0 ** -24)
        assert ((got.double() - ref).abs() <= gam * mag).all(), img
        named = {r for r in img if 0 <= r < rows}
        assert all(float(got[r].abs().max()) == 0.0 for r in range(rows) if r not in named)
        if 3 in named:  # latent 0: only the frame gradients
            assert torch.equal(got[3], latent_rows_fp32(glat, img, table, torch.zeros(rows, 32), 0.0)[3])


def test_graph_step_equals_the_eager_step_and_runs_repeat(env, monkeypatch):
    """The captured K = 4 step (repeat included) equals the eager step bit for bit over 10 steps on the same draws; two seeded
    eager runs under torch.use_deterministic_algorithms(True) repeat bit for bit."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    bboxs = [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20), (0, 32, 0, 32)]
    data, frs, images = dataset(ray_sampler, dev, 4, 32, 32, bboxs)
    ids, n, rounds = [3, 1, 3, 0], 64, 16
    lat0 = torch.randn(4, 32) * 0.1
    te, tg = _trainer(nerf, fused_train, dev, 4, False, lat0), _trainer(nerf, fused_train, dev, 4, False, lat0)
    tg.capture_images(data, 4, n, max_rounds=rounds, device_draws=False)
    g = torch.Generator(device=dev).manual_seed(13)
    for i in range(10):
        draws = torch.rand(4 * rounds * n, dtype=torch.float64, device=dev, generator=g)
        step_ids = ids if i % 2 == 0 else [2, 2, 1, 0]
        la = te.step_images(data, step_ids, n, draws=draws, max_rounds=rounds).clone()
        lb = tg.step_images_graph(torch.tensor(step_ids, dtype=torch.int32, device=dev), draws=draws).clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb), (i, la, lb)
        assert torch.equal(te.params, tg.params) and torch.equal(te.exp_avg_sq, tg.exp_avg_sq), i
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            t = _trainer(nerf, fused_train, dev, 4, True, lat0)
            torch.manual_seed(77)
            losses = [t.step_images(data, ids, n).clone() for _ in range(3)]
            torch.cuda.synchronize()
            runs.append((torch.stack(losses), t.params.clone()))
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_launches_per_step_are_the_documented_ones(env):
    """nfb_launch_count per eager step equals step_images' docstring (K = 1 and K >= 2); a graph replay issues no library call
    from the host."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    eng = _engine.renderer_for(dev)
    doc = fused_train.FusedTrainer.step_images.__doc__
    one, many = int(re.search(r"K = 1: (\d+) =", doc).group(1)), int(re.search(r"K >= 2: (\d+) =", doc).group(1))
    assert (one, many) == (16, 19)  # Adam is 2 launches (device-side schedule) in every step
    data, frs, images = dataset(ray_sampler, dev, 3, 32, 32, [(8, 24, 6, 26)] * 3)
    tr = _trainer(nerf, fused_train, dev, 3, True)
    for ids, want in (([1], one), ([0, 2], many), ([0, 1, 2, 1], many)):
        tr.step_images(data, ids, 64)  # sizes the sampler's scratch
        l0 = eng.launch_count()
        tr.step_images(data, ids, 64)
        assert eng.launch_count() - l0 == want, ids
    tr.capture_images(data, 2, 64)
    l0 = eng.launch_count()
    tr.step_images_graph([1, 2])
    torch.cuda.synchronize()
    assert eng.launch_count() == l0


def test_step_over_the_memory_budget_runs_chunked(env, monkeypatch):
    """With NFB_TRAIN_MEM_MB=48 the K = 4 step (256 rays, 64c+64f) renders and differentiates in chunks: loss and bucket agree with
    the in-budget step within the chunked path's tolerance (3e-3 of each tensor's max; each chunk has its own loss scale)."""
    nerf, _engine, fused_train, ray_sampler, dev = env
    data, frs, images = dataset(ray_sampler, dev, 3, 32, 32, [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20)])
    ids, n = [0, 2, 1, 2], 64
    draws = torch.rand(4 * 16 * n, dtype=torch.float64, device=dev)
    lat0 = torch.randn(3, 32) * 0.1
    res = []
    for budget in ("20000", "48"):
        monkeypatch.setenv("NFB_TRAIN_MEM_MB", budget)
        tr = _trainer(nerf, fused_train, dev, 3, True, lat0)
        tr._own_engine()
        sb = tr._images_buffers(data, 4, n)
        sb["img"].copy_(torch.tensor(ids, dtype=torch.int32))
        tr._images_sample(data, sb, n, draws, 16)
        torch.manual_seed(5)
        eng = _engine.renderer_for(dev)
        l0 = eng.launch_count()
        tr._images_gradients(sb, 4, n)
        torch.cuda.synchronize()
        res.append((tr.loss[:2].clone(), [t.clone() for t in tr._gviews] + [tr.grads[tr.lat_off:].clone()], eng.launch_count() - l0))
    (l1, g1, n1), (l2, g2, n2) = res
    assert n2 > n1 + 10
    assert float((l1 - l2).abs().max()) < 1e-5
    for a, b in zip(g1, g2):
        assert float((a - b).abs().max()) <= 3e-3 * max(float(a.abs().max()), 1e-12)
