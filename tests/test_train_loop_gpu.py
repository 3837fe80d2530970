"""How FusedTrainer's step paths combine over a run: the device learning-rate schedule against the reference's float64 expression,
eager and captured steps of every kind mixed on one trainer against an eager-only run bit for bit, and graphs replayed across
other work on the device's one renderer handle — bit for bit while that work grows no buffer, refused ("capture again") without
a launch once it has.

(a) nfb_adam_step_dev's lr_over_bc1 / sqrt_bc2 equal fp32(lr64(s) / (1 - b1^s)) and fp32(sqrt(1 - b2^s)) at steps 1-2,000, around
    two decay lengths and at 10^6, for three schedules: lr64 is the reference's float64 expression on the Python constants
    (train_transformed_rays.py:393-399), b1, b2 the FP32 betas the moment update uses.
(b) 2048 rays, 64c+64f, deterministic sampling (inside a graph Philox draws other numbers than a seeded eager call), 24 steps with
    the 250-step decay: graph-only, E/G alternation, step_graph / step_images_graph / step_images, and K = 4 steps mixed with K = 1
    steps each equal an eager-only trainer after every step (losses, bucket, Adam moments; gradients zero; tr.iter = the device
    step counter).
(c) Graphs captured at 2048 rays and at K = 4 x 256 replay bit for bit across validation renders, frame products, another
    trainer's steps and set_frames that fit the buffers; after each call that grows them the replays raise before any launch,
    and after capturing again the run goes on bit for bit.  A refused graph's replay is replaced by a stub that fails the test,
    so a stale graph never reaches the device."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import nerface_oracle as O
from test_train_images_gpu import dataset, make_model

pytestmark = pytest.mark.gpu

B1F, B2F = float(np.float32(0.9)), float(np.float32(0.999))
N_RAYS, ROUNDS = 2048, 16
BOXES = [(8, 56, 8, 56), (4, 60, 10, 50), (0, 64, 0, 64), (16, 48, 0, 64)]


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _capi, _engine, fused_train, ray_sampler
    return SimpleNamespace(nerf=nerf, capi=_capi, engine=_engine, fused_train=fused_train, ray_sampler=ray_sampler,
                           dev=torch.device("cuda", 0))


@pytest.fixture
def E(env, monkeypatch):
    """env with a renderer handle of the test's own: every trainer, sampler and drop-in call of the test shares it, and its buffers
    start empty, so which calls grow them does not depend on the tests that ran before."""
    eng = env.engine.Renderer(env.dev)
    monkeypatch.setitem(env.engine._renderers, ("cuda", env.dev.index), eng)
    yield SimpleNamespace(**vars(env), eng=eng)
    torch.cuda.synchronize()


def lr64(s, lr0, factor, decay):
    """The rate of 1-based step s: the reference sets lr0 * factor ** (i / decay) after the step of loop index i, so step s runs
    at exponent (s - 2) / decay, and step 1 at lr0."""
    i = s - 1
    return lr0 if i <= 0 else lr0 * factor ** ((i - 1) / decay)


def adam_state(E, lr0=5e-4, factor=0.1, decay=250.0, step=0, table_offset=-1, row=None):
    st = E.capi.NfbAdamDev(step=step, pad=0, lr0=lr0, decay_factor=factor, decay_steps=decay, beta1=0.9, beta2=0.999, eps=1e-8,
                           grad_scale=1.0, reg_weight=0.005, table_offset=table_offset, row=row, lr_over_bc1=0.0, sqrt_bc2=1.0,
                           reg_offset=-1)
    return torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8)


def read_state(E, t):
    return E.capi.NfbAdamDev.from_buffer_copy(bytes(t.cpu().numpy().tobytes()))


@pytest.mark.parametrize("lr0,factor,decay", [(5e-4, 0.1, 250000), (5e-4, 0.1, 250), (5e-4, 1.0, 250000)])
def test_device_schedule_is_the_reference_float64_expression(E, lr0, factor, decay):
    """(a) One NfbAdamDev per step s, its counter at s - 1, each advanced by one nfb_adam_step_dev on a 32-float bucket: the step's
    scalars are the float64 values rounded to FP32 once, bit for bit.  CUDA's double pow is not correctly rounded, so a value
    within an ulp of an FP32 tie could in principle round the other way; a mismatch lists both doubles."""
    steps = sorted(set(range(1, 2001)) | {d + k for d in (250, 250000) for k in range(-2, 3)} | {10 ** 6})
    states = torch.stack([adam_state(E, lr0, factor, float(decay), step=s - 1) for s in steps]).to(E.dev)  # [steps, sizeof]
    p, g, m, v = (torch.zeros(32, device=E.dev) for _ in range(4))
    for j in range(len(steps)):
        E.eng.adam_step_dev(p, g, m, v, states[j])
    got = states.cpu()
    bad = []
    for j, s in enumerate(steps):
        st = read_state(E, got[j])
        assert st.step == s and st.reg_offset == -1  # no table: no regulariser
        want_lr = lr64(s, lr0, factor, decay) / (1.0 - B1F ** s)
        want_bc = math.sqrt(1.0 - B2F ** s)
        if st.lr_over_bc1 != float(np.float32(want_lr)) or st.sqrt_bc2 != float(np.float32(want_bc)):
            bad.append((s, st.lr_over_bc1, want_lr, float(np.float32(want_lr)), st.sqrt_bc2, want_bc, float(np.float32(want_bc))))
    assert not bad, f"{len(bad)} of {len(steps)} steps (s, got lr/bc1, float64, fp32 of it, got sqrt_bc2, float64, fp32): {bad[:10]}"
    assert torch.equal(p, torch.zeros_like(p))


def test_regularised_row_comes_from_the_row_index(E):
    """(a) reg_offset = table_offset + 32 * row[0] for row >= 0; -1 for row < 0, a NULL row pointer, or no table."""
    p, g, m, v = (torch.zeros(4 * 32, device=E.dev) for _ in range(4))
    row = torch.zeros(1, device=E.dev, dtype=torch.int64)
    for r, table, ptr, want in ((2, 32, True, 96), (0, 32, True, 32), (-1, 32, True, -1), (2, 32, False, -1), (2, -1, True, -1)):
        row.fill_(r)
        st = adam_state(E, table_offset=table, row=row.data_ptr() if ptr else None).to(E.dev)
        E.eng.adam_step_dev(p, g, m, v, st)
        assert read_state(E, st).reg_offset == want, (r, table, ptr)


# ---- (b), (c): trainers on 64x64 training images, rays from the device sampler as test_one_image_step_is_the_existing_step draws them

def trainer(E, latents, prec="fast", seed=100):
    return E.fused_train.FusedTrainer(make_model(E.nerf, O.random_init_params(seed), E.dev),
                                      make_model(E.nerf, O.random_init_params(seed + 1), E.dev), n_latent=latents.shape[0], lr=5e-4,
                                      lr_decay_steps=250.0, lr_decay_factor=0.1, num_coarse=64, num_fine=64, perturb=False,
                                      noise_std=0.0, latent_reg=0.005, latent_codes=latents, precision=prec)


def training_set(E, n_images=3):
    data, frs, images = dataset(E.ray_sampler, E.dev, n_images, 64, 64, BOXES[:n_images])
    single = E.ray_sampler.RaySampler(64, 64, BOXES[:n_images], size=N_RAYS, device=E.dev)
    return data, frs, images, single


def one_image_batches(E, data, frs, images, single, steps, seed):
    """Per step: image (5i mod N), its draws, and the rays nfb_sample_rays selects with them."""
    g = torch.Generator(device=E.dev).manual_seed(seed)
    out = []
    for i in range(steps):
        img = (5 * i) % data.n_images
        draws = torch.rand(ROUNDS * N_RAYS, dtype=torch.float64, device=E.dev, generator=g)
        b = single.sample(img, draws=draws, pose=frs[img]["pose"], intrinsics=frs[img]["intrinsics"], image=images[img],
                          background=frs[0]["bg"], max_rounds=ROUNDS)
        rays = tuple(b[k].clone() for k in ("ray_origins", "ray_directions", "target"))
        out.append(dict(img=img, draws=draws, rays=rays, bg=b["background"].clone(), expr=data.expressions[img]))
    return out


def images_batches(E, data, k, n, steps, seed):
    g = torch.Generator(device=E.dev).manual_seed(seed)
    ids = [[3, 1, 3, 0], [2, 2, 1, 0], [0, 1, 2, 3]]
    return [dict(ids=ids[i % 3][:k], draws=torch.rand(k * ROUNDS * n, dtype=torch.float64, device=E.dev, generator=g))
            for i in range(steps)]


def run_step(E, t, kind, data, b1, bk, nk):
    """kind: E = step(), G = step_graph, S = step_images at K = 1, I1 = step_images_graph at K = 1, M = step_images at K,
    IK = step_images_graph at K."""
    if kind == "E":
        return t.step(*b1["rays"], b1["expr"], b1["img"], background=b1["bg"]).clone()
    if kind == "G":
        return t.step_graph(*b1["rays"], b1["expr"], b1["img"], background=b1["bg"]).clone()
    if kind == "S":
        return t.step_images(data, [b1["img"]], N_RAYS, draws=b1["draws"], max_rounds=ROUNDS).clone()
    if kind == "I1":
        return t.step_images_graph([b1["img"]], draws=b1["draws"]).clone()
    if kind == "M":
        return t.step_images(data, bk["ids"], nk, draws=bk["draws"], max_rounds=ROUNDS).clone()
    assert kind == "IK"
    return t.step_images_graph(bk["ids"], draws=bk["draws"]).clone()


def assert_same_run(E, ref, t, loss_ref, loss, what):
    """After a step: loss, parameters and Adam moments equal the reference bit for bit, the gradient bucket is zero, and the host
    step counter is the device state's."""
    assert torch.equal(loss_ref, loss), (what, loss_ref, loss)
    for name in ("params", "exp_avg", "exp_avg_sq"):
        a, b = getattr(ref, name), getattr(t, name)
        if not torch.equal(a, b):
            d = (a - b).abs()
            pytest.fail(f"{what}: {name} differs at {int((d > 0).sum())} elements, first {int(d.nonzero()[0])}, max |d| {float(d.max()):.3e}")
    assert float(t.grads.abs().max()) == 0.0, what
    assert t.iter == ref.iter == read_state(E, t._adam).step, what


@pytest.mark.parametrize("prec", ["fast", "exact"])
def test_eager_and_captured_one_image_steps_repeat_an_eager_run(E, prec):
    """(b) K = 1: graph only; E G G E G E ...; step_graph / step_images_graph / step_images in turn — each against an eager-only
    trainer fed the same rays, after every one of 24 steps."""
    data, frs, images, single = training_set(E)
    batches = one_image_batches(E, data, frs, images, single, 24, seed=4)
    lat0 = torch.randn(3, 32, generator=torch.Generator().manual_seed(2)) * 0.1
    ref = trainer(E, lat0, prec)
    runs = {"graph": "G" * 24, "alternating": "EGGEGE" * 4, "images": ["G", "I1", "S"] * 8}
    ts = {name: trainer(E, lat0, prec) for name in runs}
    for t in ts.values():
        t.capture(N_RAYS)
    ts["images"].capture_images(data, 1, N_RAYS, max_rounds=ROUNDS, device_draws=False)
    for i, b in enumerate(batches):
        loss_ref = run_step(E, ref, "E", data, b, None, None)
        losses = {name: run_step(E, t, runs[name][i], data, b, None, None) for name, t in ts.items()}
        torch.cuda.synchronize()
        for name, t in ts.items():
            assert_same_run(E, ref, t, loss_ref, losses[name], f"{prec} {name} step {i + 1} ({runs[name][i]})")
    assert int(ts["images"].shortfall.sum()) == 0


def test_several_image_steps_interleave_with_one_image_steps(E):
    """(b) K = 4 x 512 eager and captured steps between K = 1 eager and captured steps on one trainer (the regulariser moves from
    Adam to the latent-row launch and back) against the same sequence of eager steps."""
    data, frs, images, single = training_set(E, n_images=4)
    b1s = one_image_batches(E, data, frs, images, single, 24, seed=6)
    bks = images_batches(E, data, 4, 512, 24, seed=7)
    lat0 = torch.randn(4, 32, generator=torch.Generator().manual_seed(3)) * 0.1
    ref, t = trainer(E, lat0), trainer(E, lat0)
    t.capture_images(data, 4, 512, max_rounds=ROUNDS, device_draws=False)  # the larger sampler scratch first
    t.capture(N_RAYS)
    plan = ["M", "IK", "E", "IK", "G", "M", "G", "IK", "M", "E", "G", "IK"] * 2
    for i, kind in enumerate(plan):
        loss_ref = run_step(E, ref, "M" if kind in ("M", "IK") else "E", data, b1s[i], bks[i], 512)
        loss = run_step(E, t, kind, data, b1s[i], bks[i], 512)
        torch.cuda.synchronize()
        assert_same_run(E, ref, t, loss_ref, loss, f"step {i + 1} ({kind})")


def test_graphs_replay_across_other_work_and_refuse_after_growth(E, monkeypatch):
    """(c) Graphs at 2048 rays and K = 4 x 256 replay bit for bit across work that grows nothing, and the buffer epoch stays; each
    growing call (another trainer's 4096-ray step, set_frames with 5 frames, a K = 8 step) bumps it, the next replay of either
    graph raises before any launch, and after capturing again the run continues bit for bit."""
    nerf, eng = E.nerf, E.eng
    data, frs, images, single = training_set(E, n_images=4)
    b1s = one_image_batches(E, data, frs, images, single, 12, seed=8)
    bks = images_batches(E, data, 4, 256, 12, seed=9)
    lat0 = torch.randn(4, 32, generator=torch.Generator().manual_seed(5)) * 0.1
    plan = ["G", "IK"] * 6

    def capture(t):
        t.capture(N_RAYS)
        t.capture_images(data, 4, 256, max_rounds=ROUNDS, device_draws=False)

    # the uninterrupted run
    tu = trainer(E, lat0)
    capture(tu)
    snaps = []
    for i, kind in enumerate(plan):
        loss = run_step(E, tu, kind, data, b1s[i], bks[i], 256)
        snaps.append(SimpleNamespace(loss=loss, params=tu.params.clone(), exp_avg=tu.exp_avg.clone(), exp_avg_sq=tu.exp_avg_sq.clone(),
                                     iter=tu.iter))

    ti, other = trainer(E, lat0), trainer(E, lat0 * 2, seed=200)
    capture(ti)
    epoch = eng.buffer_epoch()
    assert ti._graph["epoch"] == ti._igraph["epoch"] == epoch

    def replay(i):
        loss = run_step(E, ti, plan[i], data, b1s[i], bks[i], 256)
        torch.cuda.synchronize()
        assert_same_run(E, snaps[i], ti, snaps[i].loss, loss, f"step {i + 1} ({plan[i]})")

    # ---- work that grows nothing
    fr = O.synthetic_frame(1, 512, 512)
    ro, rd = O.ray_bundle(512, 512, fr["intrinsics"], fr["pose"])
    vblk = dict(num_coarse=64, num_fine=64, perturb=False, lindisp=False, radiance_field_noise_std=0.0, white_background=False,
                chunksize=65536)
    vcfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, validation=vblk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    pin = lambda t: t.contiguous().pin_memory()  # noqa: E731
    fh = O.synthetic_frame(2, 128, 128)
    host = dict(expr=pin(fh["expr"]), latent=pin(fh["latent"]), bg=pin(fh["bg"].reshape(-1, 3)),
                out=torch.empty(11 * 128 * 128).pin_memory())

    def validation():
        with torch.no_grad():
            out = nerf.run_one_iter_of_nerf(512, 512, fr["intrinsics"], ti.mc, ti.mf, ro.to(E.dev), rd.to(E.dev), vcfg,
                                            mode="validation", expressions=data.expressions[1], background_prior=fr["bg"].to(E.dev),
                                            latent_code=ti.latent_codes[1])
        assert torch.isfinite(out[3]).all()

    def frame_host_and_products():
        eng.render_frame_host(fh["pose"], fh["intrinsics"], 128, 128, 0, 128, 0.2, 0.8, host["expr"], host["latent"], host["bg"], 64,
                              64, host["out"])
        torch.cuda.synchronize()
        o, n = host["out"].to(E.dev), 128 * 128
        u8 = E.ray_sampler.frame_products(o[5 * n:8 * n].view(128, 128, 3), o[8 * n:9 * n].view(128, 128),
                                          o[10 * n:11 * n].view(128, 128), fh["intrinsics"], want_disparity=True)
        assert u8[0].shape == (128, 128, 3)

    work = [validation,
            frame_host_and_products,
            lambda: other.step(*[r[:1536] for r in b1s[5]["rays"]], b1s[5]["expr"], 2, background=b1s[5]["bg"][:1536]),
            lambda: eng.set_frames(data.expressions, other.latent_codes),
            lambda: other.step_images(data, [1, 2, 1], 256, max_rounds=ROUNDS),
            lambda: eng.set_frames(data.expressions[:2], other.latent_codes[:2])]
    for i, w in enumerate(work):
        replay(i)
        w()
    assert eng.buffer_epoch() == epoch

    # ---- calls that grow the handle's buffers
    fr64 = O.synthetic_frame(3, 64, 64)
    ro64, rd64 = (x.reshape(-1, 3).to(E.dev) for x in O.ray_bundle(64, 64, fr64["intrinsics"], fr64["pose"]))
    tgt64 = torch.rand(4096, 3, generator=torch.Generator().manual_seed(6)).to(E.dev)
    grow = [("another trainer's 4096-ray step",
             lambda: other.step(ro64, rd64, tgt64, data.expressions[0], 0, background=fr64["bg"].reshape(-1, 3).to(E.dev))),
            ("set_frames with 5 frames", lambda: eng.set_frames(torch.cat([data.expressions, data.expressions[:1]]),
                                                                torch.cat([other.latent_codes, other.latent_codes[:1]]))),
            ("a K = 8 step", lambda: other.step_images(data, [0, 1, 2, 3, 3, 2, 1, 0], 256, max_rounds=ROUNDS))]
    i = len(work)

    def stale(*args, **kwargs):
        pytest.fail("a graph whose buffers were re-allocated reached replay()")

    for what, g in grow:
        assert eng.buffer_epoch() == ti._graph["epoch"] == ti._igraph["epoch"], what
        g()
        torch.cuda.synchronize()
        monkeypatch.setattr(ti._graph["graph"], "replay", stale)
        monkeypatch.setattr(ti._igraph["graph"], "replay", stale)
        launches, it = eng.launch_count(), ti.iter
        with pytest.raises(RuntimeError, match="capture again"):
            run_step(E, ti, "G", data, b1s[i], bks[i], 256)
        with pytest.raises(RuntimeError, match="capture again"):
            run_step(E, ti, "IK", data, b1s[i], bks[i], 256)
        assert eng.launch_count() == launches and ti.iter == it, what
        assert eng.buffer_epoch() > ti._graph["epoch"], what
        capture(ti)
        for _ in range(2):
            replay(i)
            i += 1
    assert i == len(plan)
