"""The fused training step (nerf/fused_train.py: loss gradient, backward into a flat bucket, Adam + zero_grad, re-pack — all
libnfb launches) against the path the unmodified train script takes: run_one_iter_of_nerf + torch mse_loss + loss.backward()
+ torch.optim.Adam + the script's LR schedule (train_transformed_rays.py:336-400)."""
import pytest
import torch

import nerface_oracle as O

pytestmark = pytest.mark.gpu


def make_model(nerf, params, dev):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params)
    return m.to(dev)


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train
    return nerf, _engine, fused_train, torch.device("cuda", 0)


def _batches(dev, steps, n):
    H = W = 32
    fr = O.synthetic_frame(2, H, W)
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev)
    bg = fr["bg"].reshape(-1, 3).to(dev)
    g = torch.Generator().manual_seed(3)
    tgt = torch.rand(H * W, 3, generator=g).to(dev)
    idx = [torch.randperm(H * W, generator=g)[:n].to(dev) for _ in range(steps)]
    return fr, ro, rd, bg, tgt, idx


def test_fused_step_matches_the_reference_style_step(env):
    """From identical state and identical noise: (a) the fused step's gradient bucket equals the gradients loss.backward()
    leaves on the drop-in path (1e-6 of each tensor's largest entry), (b) after the optimizer step every parameter agrees to
    1e-6, (c) over 10 steps the two loss curves agree to 2e-6.

    Longer parameter trajectories are NOT compared element-wise: with random-init (96 % transparent) volumes a fifth of the
    gradient entries are below Adam's eps = 1e-8, where the update is lr * g / eps — a gain of 5e4 on the ~1e-11 absolute noise
    that the order of the weight-gradient atomics leaves in g.  Two runs of the SAME loop differ by > 1e-6 in 3 % of the
    parameters after 5 steps (measured, DESIGN.md 6); the optimizer arithmetic itself is pinned by
    test_adam_kernel_matches_torch_adam on identical gradients."""
    nerf, _engine, fused_train, dev = env
    from nerf._engine import PARAM_ORDER
    steps, n, lat = 10, 64, 3
    fr, ro, rd, bg, tgt, idx = _batches(dev, steps, n)
    expr = fr["expr"].to(dev)
    lr0, decay, factor = 5e-4, 250.0, 0.1  # a short decay so the schedule matters within 10 steps
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False, chunksize=2048)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))

    # ---- reference-style loop on the drop-in API (train_transformed_rays.py:336-400)
    mc, mf = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
    latent_codes = torch.zeros(8, 32, device=dev, requires_grad=True)
    opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()) + [latent_codes], lr=lr0)
    ref_losses, ref_grads, ref_params1 = [], None, None
    for i in range(steps):
        sel = idx[i]
        torch.manual_seed(1000 + i)
        out = nerf.run_one_iter_of_nerf(32, 32, fr["intrinsics"], mc, mf, ro[sel], rd[sel], cfg, mode="train", expressions=expr,
                                        background_prior=bg[sel], latent_code=latent_codes[lat])
        coarse = torch.nn.functional.mse_loss(out[0], tgt[sel])
        fine = torch.nn.functional.mse_loss(out[3], tgt[sel])
        loss = coarse + fine + torch.norm(latent_codes[lat]) * 0.0005 * 10
        loss.backward()
        if i == 0:
            ref_grads = [[dict(m.named_parameters())[k].grad for k in PARAM_ORDER] for m in (mc, mf)]
            ref_grads = [[g.clone() if g is not None else None for g in gs] for gs in ref_grads] + [latent_codes.grad[lat].clone()]
        opt.step()
        opt.zero_grad()
        for gp in opt.param_groups:  # train_transformed_rays.py:393-399
            gp["lr"] = lr0 * factor ** (i / decay)
        if i == 0:
            ref_params1 = [p.detach().clone() for p in list(mc.parameters()) + list(mf.parameters())] + [latent_codes.detach().clone()]
        ref_losses.append((float(coarse.detach()), float(fine.detach())))

    # ---- fused loop, same inputs, same noise stream
    mc2, mf2 = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
    tr = fused_train.FusedTrainer(mc2, mf2, n_latent=8, lr=lr0, lr_decay_steps=decay, lr_decay_factor=factor, num_coarse=64,
                                  num_fine=64, perturb=True, noise_std=0.1, near=0.2, far=0.8, latent_reg=0.005)
    eng = _engine.renderer_for(dev)
    # (a) gradients of step 0, taken before the optimizer consumes (and zeroes) them
    sel = idx[0]
    torch.manual_seed(1000)
    noise = tr._draw_noise(n)
    eng.set_frame(expr, tr.latent_codes[lat])
    o = eng.render(ro[sel], rd[sel], 0.2, 0.8, 64, 64, perturb=True, noise_std=0.1, background=bg[sel], noise=noise, train=True)
    g0, g1 = torch.empty((n, 3), device=dev), torch.empty((n, 3), device=dev)
    tr.loss.zero_()
    eng.loss_mse_grad(o["rgb_coarse"], o["rgb_fine"], tgt[sel].contiguous(), n, g0, g1, tr.loss)
    glat = tr.grads[tr.lat_off + 32 * lat:tr.lat_off + 32 * lat + 32]
    eng.backward_into((g0, None, None, g1, None, None, None), tr._pc, tr._pf, tr._gc, tr._gf, glat)
    torch.cuda.synchronize()
    for gs_ref, gs in zip(ref_grads[:2], (tr._gc, tr._gf)):
        for k, a, b in zip(PARAM_ORDER, gs_ref, gs):
            assert (a is None) == (b is None), k
            if a is not None:
                assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-12), k
    assert float((ref_grads[2] - glat).abs().max()) <= 1e-6 * float(ref_grads[2].abs().max())
    assert abs(float(tr.loss[0]) - ref_losses[0][0]) < 2e-6 and abs(float(tr.loss[1]) - ref_losses[0][1]) < 2e-6
    tr.grads.zero_()

    fused_losses = []
    for i in range(steps):
        sel = idx[i]
        torch.manual_seed(1000 + i)
        lv = tr.step(ro[sel], rd[sel], tgt[sel], expr, lat, background=bg[sel])
        fused_losses.append(tuple(float(v) for v in lv))
        if i == 0:  # (b) one optimizer step from identical state
            torch.cuda.synchronize()
            worst = max(float((p - q.detach()).abs().max()) for p, q in zip(
                ref_params1, list(mc2.parameters()) + list(mf2.parameters()) + [tr.latent_codes]))
            print(f"fused vs drop-in + torch.optim.Adam after one step: max|d param| = {worst:.3e}")
            assert worst <= 1e-6
    torch.cuda.synchronize()
    for (a, b), (c, d) in zip(ref_losses, fused_losses):  # (c)
        assert abs(a - c) < 2e-6 and abs(b - d) < 2e-6, (a, c, b, d)
    worst = max(float((p.detach() - q.detach()).abs().max()) for p, q in zip(
        list(mc.parameters()) + list(mf.parameters()), list(mc2.parameters()) + list(mf2.parameters())))
    assert worst <= 2.5 * steps * lr0  # no parameter ran away
    assert float(tr.latent_codes[lat].abs().max()) > 0 and float(tr.latent_codes[lat + 1].abs().max()) == 0.0
    # the models' parameters ARE the bucket: a validation render through the drop-in API sees the trained weights without a re-pack
    vcfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, validation=dict(blk, perturb=False, radiance_field_noise_std=0.0)),
                             dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    with torch.no_grad():
        l0 = eng.launch_count()
        a = nerf.run_one_iter_of_nerf(32, 32, fr["intrinsics"], mc2, mf2, ro[:64], rd[:64], vcfg, mode="validation", expressions=expr,
                                      background_prior=bg[:64], latent_code=tr.latent_codes[lat])
        assert eng.launch_count() - l0 == 2  # frame fold + render: no weight re-pack
        assert all(torch.isfinite(t).all() for t in a)


def test_adam_kernel_matches_torch_adam(env):
    """nfb_adam_step against torch.optim.Adam on identical gradients over 10 steps: flat bucket, gradient magnitudes from 1e-12
    to 1, the reference's LR schedule, and the latent regulariser on one 32-float row (as an explicit loss term on the torch side)."""
    nerf, _engine, fused_train, dev = env
    eng = _engine.renderer_for(dev)
    g = torch.Generator().manual_seed(11)
    n, row = 256 * 40 + 64, 256 * 40 + 32
    p0 = ((torch.rand(n, generator=g) - 0.5) * 0.2).to(dev)
    p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=5e-4)
    p, m, v = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    lr0, decay, factor = 5e-4, 250.0, 0.1
    for i in range(10):
        mag = 10.0 ** (torch.rand(n, generator=g) * 12.0 - 12.0)
        grad = ((torch.rand(n, generator=g) - 0.5) * 2.0 * mag).to(dev)
        grad[:100] = 0.0  # elements that never receive a gradient must not move
        lr_i = lr0 if i == 0 else lr0 * factor ** ((i - 1) / decay)
        for gp in opt.param_groups:
            gp["lr"] = lr_i
        opt.zero_grad()
        reg = torch.norm(p_ref[row:row + 32]) * 0.005
        reg.backward()
        p_ref.grad += grad
        opt.step()
        gbuf = grad.clone()
        eng.adam_step(p, gbuf, m, v, lr_i, i + 1, reg_offset=row, reg_weight=0.005)
        assert float(gbuf.abs().max()) == 0.0  # zero_grad fused
    torch.cuda.synchronize()
    d = (p - p_ref.detach()).abs()
    print(f"adam kernel vs torch.optim.Adam, 10 steps: max|d| = {float(d.max()):.3e}")
    assert float(d.max()) <= 1e-6
    assert torch.equal(p[:100], p0[:100])


def test_adam_dev_kernel_matches_torch_adam(env):
    """nfb_adam_step_dev — step counter, the reference's LR schedule and the regularised row in an NfbAdamDev on the device —
    against torch.optim.Adam over the same 10 steps as test_adam_kernel_matches_torch_adam (gradients from 1e-12 to 1, the latent
    regulariser on one 32-float row); the state ends at step 10 with that row as its regularised offset."""
    from nerf import _capi
    nerf, _engine, fused_train, dev = env
    eng = _engine.renderer_for(dev)
    g = torch.Generator().manual_seed(11)
    n, row = 256 * 40 + 64, 256 * 40 + 32
    p0 = ((torch.rand(n, generator=g) - 0.5) * 0.2).to(dev)
    p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=5e-4)
    p, m, v = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    lr0, decay, factor = 5e-4, 250.0, 0.1
    row_index = torch.full((1,), 1, device=dev, dtype=torch.int64)  # the table starts one row before the regularised one
    st = _capi.NfbAdamDev(step=0, pad=0, lr0=lr0, decay_factor=factor, decay_steps=decay, beta1=0.9, beta2=0.999, eps=1e-8,
                          grad_scale=1.0, reg_weight=0.005, table_offset=row - 32, row=row_index.data_ptr(), lr_over_bc1=0.0,
                          sqrt_bc2=1.0, reg_offset=-1)
    dev_state = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(dev)
    for i in range(10):
        mag = 10.0 ** (torch.rand(n, generator=g) * 12.0 - 12.0)
        grad = ((torch.rand(n, generator=g) - 0.5) * 2.0 * mag).to(dev)
        grad[:100] = 0.0
        for gp in opt.param_groups:
            gp["lr"] = lr0 if i == 0 else lr0 * factor ** ((i - 1) / decay)
        opt.zero_grad()
        reg = torch.norm(p_ref[row:row + 32]) * 0.005
        reg.backward()
        p_ref.grad += grad
        opt.step()
        gbuf = grad.clone()
        eng.adam_step_dev(p, gbuf, m, v, dev_state)
        assert float(gbuf.abs().max()) == 0.0
    torch.cuda.synchronize()
    got = _capi.NfbAdamDev.from_buffer_copy(bytes(dev_state.cpu().numpy().tobytes()))
    assert got.step == 10 and got.reg_offset == row
    d = (p - p_ref.detach()).abs()
    print(f"device-state adam kernel vs torch.optim.Adam, 10 steps: max|d| = {float(d.max()):.3e}")
    assert float(d.max()) <= 1e-6
    assert torch.equal(p[:100], p0[:100])


def test_fused_step_launch_budget(env):
    """After the backward: Adam (+ zero_grad) is one launch and the re-pack two (FP64 fold, pack) — 3 in all; the whole step stays
    under 20 launches."""
    nerf, _engine, fused_train, dev = env
    fr, ro, rd, bg, tgt, idx = _batches(dev, 3, 64)
    mc, mf = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
    tr = fused_train.FusedTrainer(mc, mf, n_latent=4)
    eng = _engine.renderer_for(dev)
    expr = fr["expr"].to(dev)
    tr.step(ro[idx[0]], rd[idx[0]], tgt[idx[0]], expr, 1, background=bg[idx[0]])
    l0 = eng.launch_count()
    tr.step(ro[idx[1]], rd[idx[1]], tgt[idx[1]], expr, 1, background=bg[idx[1]])
    total = eng.launch_count() - l0
    l1 = eng.launch_count()
    eng.adam_step(tr.params, tr.grads, tr.exp_avg, tr.exp_avg_sq, 1e-4, 3)
    eng.repack(tr._pc, tr._pf)
    assert eng.launch_count() - l1 == 3
    assert total <= 20, total


def test_in_loop_validation_keeps_the_saved_training_state(env):
    """train_transformed_rays.py:427-504 renders validation frames under no_grad between optimizer steps; a no_grad render
    between a training forward and its backward must not disturb the state the backward consumes."""
    nerf, _engine, fused_train, dev = env
    fr, ro, rd, bg, tgt, idx = _batches(dev, 2, 64)
    expr = fr["expr"].to(dev)
    blk = dict(num_coarse=64, num_fine=64, perturb=False, lindisp=False, radiance_field_noise_std=0.0, white_background=False, chunksize=2048)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk, validation=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    grads = []
    for interleave in (False, True):
        mc, mf = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
        lat = torch.full((32,), 0.01, device=dev, requires_grad=True)
        out = nerf.run_one_iter_of_nerf(32, 32, fr["intrinsics"], mc, mf, ro[idx[0]], rd[idx[0]], cfg, mode="train", expressions=expr,
                                        background_prior=bg[idx[0]], latent_code=lat)
        if interleave:
            with torch.no_grad():
                nerf.run_one_iter_of_nerf(32, 32, fr["intrinsics"], mc, mf, ro[:128], rd[:128], cfg, mode="validation", expressions=expr * 0.5,
                                          background_prior=bg[:128], latent_code=torch.zeros(32, device=dev))
        loss = ((out[0] - tgt[idx[0]]) ** 2).mean() + ((out[3] - tgt[idx[0]]) ** 2).mean()
        loss.backward()
        grads.append([p.grad.clone() for p in mc.parameters() if p.grad is not None] + [lat.grad.clone()])
    for a, b in zip(*grads):
        assert float((a - b).abs().max()) <= 1e-6 * max(1.0, float(a.abs().max()))


def test_training_over_the_memory_budget_runs_in_chunks(env, monkeypatch):
    """ADVICE r1: a training-mode call whose per-tile records exceed the budget (a full frame with gradients enabled needs
    hundreds of GiB) must not die in cudaMalloc.  With NFB_TRAIN_MEM_MB=48 a 160-ray batch (64c+64f: 240 tiles = 240 MiB of
    records) is processed in 5 chunks; outputs are identical and the gradients agree with the one-launch path to the FP16
    operand precision (each chunk has its own loss scale)."""
    nerf, _engine, fused_train, dev = env
    fr, ro, rd, bg, tgt, idx = _batches(dev, 1, 160)
    sel = idx[0]
    expr = fr["expr"].to(dev)
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False, chunksize=64)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    results = []
    for budget in (None, "48"):
        if budget:
            monkeypatch.setenv("NFB_TRAIN_MEM_MB", budget)
        mc, mf = make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev)
        lat = torch.full((32,), 0.01, device=dev, requires_grad=True)
        torch.manual_seed(9)
        eng = _engine.renderer_for(dev)
        l0 = eng.launch_count()
        out = nerf.run_one_iter_of_nerf(32, 32, fr["intrinsics"], mc, mf, ro[sel], rd[sel], cfg, mode="train", expressions=expr,
                                        background_prior=bg[sel], latent_code=lat)
        loss = ((out[0] - tgt[sel]) ** 2).mean() + ((out[3] - tgt[sel]) ** 2).mean() + out[6].mean() * 0.1
        loss.backward()
        torch.cuda.synchronize()
        results.append(([o.detach().clone() for o in out], [p.grad.clone() for p in list(mc.parameters()) + list(mf.parameters()) if p.grad is not None] + [lat.grad.clone()],
                        eng.launch_count() - l0))
    monkeypatch.delenv("NFB_TRAIN_MEM_MB")
    (o1, g1, n1), (o2, g2, n2) = results
    assert n2 > n1 + 10  # several chunks' worth of launches
    for a, b in zip(o1, o2):
        assert float((a - b).abs().max()) < 1e-5   # the evaluation kernel renders what the training forward renders
    for a, b in zip(g1, g2):
        assert float((a - b).abs().max()) <= 3e-3 * max(float(a.abs().max()), 1e-12)


def test_captured_graph_step_matches_the_eager_fused_step(env):
    """FusedTrainer.capture(): the whole iteration (frame fold, noise draws, SAVE forward, loss, backward, Adam with device-side
    step / LR schedule / regularised row, re-pack) replayed as ONE CUDA graph follows the eager fused loop: same losses, same
    parameters after one step (to 1e-6; later steps are chaotic at |g| < eps, see above), device step counter in lock-step.
    Deterministic sampling here: inside a graph torch's Philox offsets advance per replay, not per call, so a seeded replay does
    not draw the numbers the seeded eager calls draw (same distribution); the stochastic graph is exercised at the end."""
    nerf, _engine, fused_train, dev = env
    steps, n, lat = 4, 64, 2
    fr, ro, rd, bg, tgt, idx = _batches(dev, steps, n)
    expr = fr["expr"].to(dev)
    mk = lambda: fused_train.FusedTrainer(  # noqa: E731
        make_model(nerf, O.random_init_params(100), dev), make_model(nerf, O.random_init_params(101), dev),  # noqa: E731
                                          n_latent=8, lr=5e-4, lr_decay_steps=250.0, lr_decay_factor=0.1, num_coarse=64, num_fine=64,
                                          perturb=noisy, noise_std=0.1 if noisy else 0.0)
    noisy = False
    ta, tb = mk(), mk()
    tb.capture(n)
    eng = _engine.renderer_for(dev)
    for i in range(steps):
        sel = idx[i]
        torch.manual_seed(500 + i)
        la = ta.step(ro[sel], rd[sel], tgt[sel], expr, lat, background=bg[sel]).clone()
        torch.manual_seed(500 + i)
        tb._own_engine()  # two trainers alternate on the device's one renderer here: ta's step left ITS weights packed
        l0 = eng.launch_count()
        lb = tb.step_graph(ro[sel], rd[sel], tgt[sel], expr, lat, background=bg[sel]).clone()
        torch.cuda.synchronize()
        assert eng.launch_count() == l0  # no library call outside the graph
        assert float((la - lb).abs().max()) < 2e-6, (i, la, lb)
        if i == 0:
            assert float((ta.params - tb.params).abs().max()) <= 1e-6
    import ctypes as C
    from nerf import _capi
    st = _capi.NfbAdamDev.from_buffer_copy(bytes(tb._graph["sb"]["adam"].cpu().numpy().tobytes()))
    assert st.step == steps == tb.iter and st.reg_offset == tb.lat_off + 32 * lat
    lr_expected = 5e-4 * 0.1 ** ((steps - 2) / 250.0)
    bc1 = 1.0 - 0.9 ** steps
    assert abs(st.lr_over_bc1 - lr_expected / bc1) < 1e-9
    assert float(tb.latent_codes[lat].abs().max()) > 0 and float(tb.latent_codes[lat + 1].abs().max()) == 0.0
    noisy = True
    tc = mk()
    tc.capture(n)
    ls = [tc.step_graph(ro[idx[i]], rd[idx[i]], tgt[idx[i]], expr, lat, background=bg[idx[i]]).clone() for i in range(steps)]
    torch.cuda.synchronize()
    assert all(torch.isfinite(v).all() and 0.01 < float(v.sum()) < 1.0 for v in ls)
    assert float((ls[0] - ls[1]).abs().max()) > 0  # fresh noise on every replay
