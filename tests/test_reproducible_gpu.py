"""The fused path repeats bit for bit (include/nfb.h): identical calls give identical forward outputs, gradients and losses, so
seeded training and fitting loops follow identical trajectories, and torch.use_deterministic_algorithms(True) holds for it.

Production sizes throughout: 2048 rays at 64c+64f, the opaque-stress weights (compositing and resampling see opaque rays),
stratified sampling, sigma noise 0.1 and a background, in both precision modes."""
import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_fp64_gpu import E, FAR, NAMES, NEAR, PRECS, make_case, model, out_grads, train_forward  # noqa: F401

pytestmark = pytest.mark.gpu

N = 2048
ALL_INPUTS = ["ray_origins", "ray_directions", "expression", "background", "dir_z"]


def _params(c):
    pc = [dict(c.mc.named_parameters())[k] for k in TR.PARAM_ORDER]
    pf = [dict(c.mf.named_parameters())[k] for k in TR.PARAM_ORDER] if c.mf is not None else None
    return pc, pf


def _backward(E, c, gouts, want_params, want_latent, inputs):
    """Every tensor one backward call returns, in a fixed order."""
    pc, pf = _params(c)
    gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_latent=want_latent, want_params=want_params, inputs=inputs)
    torch.cuda.synchronize()
    named = [(f"coarse/{i}", g) for i, g in enumerate(gc or []) if g is not None]
    named += [(f"fine/{i}", g) for i, g in enumerate(gf or []) if g is not None]
    if gl is not None:
        named.append(("latent", gl))
    named += sorted(ing.items())
    return named


def _outputs(out):
    return [(k, out[k].clone()) for k in NAMES if k in out]


def _assert_equal(a, b, tag):
    assert [k for k, _ in a] == [k for k, _ in b], tag
    for (k, x), (_, y) in zip(a, b):
        assert bool(torch.isfinite(x).all()), (tag, k, "non-finite")
        assert torch.equal(x, y), (tag, k, float((x - y).abs().max()))


VARIANTS = {  # name: (rays, coarse, fine, case options, parameter gradients, latent gradient, inputs)
    "full": (N, 64, 64, dict(dir_z=True), True, True, ALL_INPUTS),
    "coarse_only": (N, 64, 0, dict(dir_z=True), True, True, ALL_INPUTS),
    "512_samples": (256, 256, 256, dict(dir_z=True), True, True, ALL_INPUTS),
    "white_bkgd": (N, 64, 64, dict(white=True, bg=False, dir_z=True), True, True, ["ray_origins", "ray_directions", "expression", "dir_z"]),
    "input_only_pe": (N, 64, 64, dict(dir_z=True), False, True, ALL_INPUTS),  # the PE-only weight-gradient launch
    "input_only_rays": (N, 64, 64, dict(dir_z=True), False, False, ["ray_origins", "ray_directions", "background", "dir_z"]),
    "chunked": (N, 64, 64, dict(dir_z=True), True, True, ALL_INPUTS),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_repeated_backward_is_bit_identical(E, variant, prec, monkeypatch):
    """One training forward, three backward calls with all output gradients non-zero: every gradient is equal across the calls.
    A second forward of the same inputs gives equal outputs and equal gradients again."""
    n, nc, nf, opts, want_params, want_latent, inputs = VARIANTS[variant]
    if variant == "chunked":
        monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")  # 16 units (32 rays) per chunk: 64 chunks, each with its own reduction
    c = make_case(E, n, nc, nf, prec, seed=31, **opts)
    out1 = _outputs(train_forward(E, c))
    gouts = out_grads(E, c, seed=32)
    runs = [_backward(E, c, gouts, want_params, want_latent, inputs) for _ in range(3)]
    assert len(runs[0]) >= len(inputs) + (1 if want_latent else 0) + (24 * (2 if nf else 1) if want_params else 0)
    for i in (1, 2):
        _assert_equal(runs[0], runs[i], f"{variant} {prec} backward {i}")
    out2 = _outputs(train_forward(E, c))
    _assert_equal(out1, out2, f"{variant} {prec} forward")
    _assert_equal(runs[0], _backward(E, c, gouts, want_params, want_latent, inputs), f"{variant} {prec} second forward")


@pytest.mark.parametrize("prec", PRECS)
def test_output_gradient_scaling_is_exact(E, prec):
    """The loss scale is a power of two chosen from max |d raw|, and every reduction runs in a fixed order: scaling the output
    gradients by 2^k scales every gradient by exactly 2^k."""
    c = make_case(E, N, 64, 64, prec, seed=33, dir_z=True)
    train_forward(E, c)
    gouts = out_grads(E, c, seed=34)
    base = _backward(E, c, gouts, True, True, ALL_INPUTS)
    tiny = torch.finfo(torch.float32).tiny
    for k in (20, -20):
        got = _backward(E, c, [g * 2.0 ** k for g in gouts], True, True, ALL_INPUTS)
        for (name, a), (_, b) in zip(base, got):
            for t in (a, b):
                assert bool(torch.isfinite(t).all()), (k, name)
                assert not bool(((t != 0) & (t.abs() < tiny)).any()), (k, name, "subnormal")
            assert torch.equal(b, a * 2.0 ** k), (k, name, float((b - a * 2.0 ** k).abs().max()))


# ------------------------------------------------------------------------------------------------ training loops
def _fresh_models(E):
    """Models with their own parameter storage (a FusedTrainer turns its models' parameters into views of its bucket)."""
    return model(E, 100, True, O.random_init_params(100, True)), model(E, 101, True, O.random_init_params(101, True))


def _batches(E, steps, seed):
    g = torch.Generator().manual_seed(seed)
    total = E.ro.shape[0]
    idx = [torch.randperm(total, generator=g)[:N].to(E.dev) for _ in range(steps)]
    return idx, torch.rand(total, 3, generator=g).to(E.dev)


def _trainer(E, prec):
    from nerf import fused_train
    mc, mf = _fresh_models(E)
    lat0 = (torch.rand(4, 32, generator=torch.Generator().manual_seed(5)) - 0.5) * 0.1
    return fused_train.FusedTrainer(mc, mf, n_latent=4, num_coarse=64, num_fine=64, perturb=True, noise_std=0.1, near=NEAR, far=FAR,
                                    precision=prec, latent_codes=lat0)


def _state(t, loss):
    return [("loss", loss.clone()), ("params", t.params.clone()), ("exp_avg", t.exp_avg.clone()),
            ("exp_avg_sq", t.exp_avg_sq.clone()), ("latent", t.latent_codes.clone())]


@pytest.mark.parametrize("prec", PRECS)
def test_fused_training_repeats(E, prec):
    """Two FusedTrainers from identical weights, 20 eager steps, re-seeded before each: losses, parameters, Adam moments and the
    latent table are equal after every step."""
    steps = 20
    idx, tgt = _batches(E, steps, 41)
    ta, tb = _trainer(E, prec), _trainer(E, prec)
    for i in range(steps):
        s = idx[i]
        states = []
        for t in (ta, tb):
            torch.manual_seed(700 + i)
            loss = t.step(E.ro[s], E.rd[s], tgt[s], E.expr, i % 4, background=E.bg[s])
            states.append(_state(t, loss))
        torch.cuda.synchronize()
        _assert_equal(states[0], states[1], f"eager {prec} step {i}")


@pytest.mark.parametrize("prec", PRECS)
def test_captured_training_repeats(E, prec):
    """The same through capture() / step_graph(): the noise is drawn inside each graph from torch's graph-safe Philox state,
    which a replay takes from the generator's seed and offset at that moment, so re-seeding before each replay gives both
    graphs the same draws."""
    steps = 20
    idx, tgt = _batches(E, steps, 42)
    ta, tb = _trainer(E, prec), _trainer(E, prec)
    ta.capture(N)
    tb.capture(N)
    for i in range(steps):
        s = idx[i]
        states = []
        for t in (ta, tb):
            torch.manual_seed(900 + i)
            loss = t.step_graph(E.ro[s], E.rd[s], tgt[s], E.expr, i % 4, background=E.bg[s])
            states.append(_state(t, loss))
        torch.cuda.synchronize()
        _assert_equal(states[0], states[1], f"captured {prec} step {i}")
    assert float(states[0][0][1].sum()) > 0.0


# ------------------------------------------------------------------------------------------------ torch's deterministic mode
@pytest.fixture
def deterministic():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


@pytest.fixture
def precision():
    from nerf import _engine
    was = _engine.get_precision()
    yield _engine.set_precision
    _engine.set_precision(was)


def _cfg(nerf):
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=N)
    return nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=NEAR, far=FAR)))


def _reference_style_training(E, steps, idx, tgt, fr):
    """run_one_iter_of_nerf in train mode, mse + latent norm, loss.backward(), torch.optim.Adam."""
    nerf = E.nerf
    mc, mf = _fresh_models(E)
    lat = ((torch.rand(4, 32, generator=torch.Generator().manual_seed(5)) - 0.5) * 0.1).to(E.dev).requires_grad_(True)
    opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()) + [lat], lr=5e-4)
    cfg = _cfg(nerf)
    losses = []
    for i in range(steps):
        s = idx[i]
        torch.manual_seed(300 + i)
        out = nerf.run_one_iter_of_nerf(48, 48, fr["intrinsics"], mc, mf, E.ro[s], E.rd[s], cfg, mode="train", expressions=E.expr,
                                        background_prior=E.bg[s], latent_code=lat[i % 4])
        loss = (torch.nn.functional.mse_loss(out[0], tgt[s]) + torch.nn.functional.mse_loss(out[3], tgt[s])
                + torch.norm(lat[i % 4]) * 0.0005 * 10)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    torch.cuda.synchronize()
    return ([(f"p{j}", p.detach().clone()) for j, p in enumerate(list(mc.parameters()) + list(mf.parameters()))]
            + [("latent", lat.detach().clone()), ("losses", torch.stack(losses))])


def _fitting(E, steps, idx, tgt, fr):
    """Frozen networks; the expression and the camera pose require grad (input-only backward through the public API)."""
    nerf = E.nerf
    mc, mf = _fresh_models(E)
    for m in (mc, mf):
        m.requires_grad_(False)
    pose = fr["pose"].to(E.dev).clone().requires_grad_(True)
    expr = E.expr.clone().requires_grad_(True)
    opt = torch.optim.Adam([pose, expr], lr=1e-3)
    cfg = _cfg(nerf)
    losses = []
    for i in range(steps):
        s = idx[i]
        torch.manual_seed(500 + i)
        ro, rd = nerf.get_ray_bundle(48, 48, fr["intrinsics"], pose)
        out = nerf.run_one_iter_of_nerf(48, 48, fr["intrinsics"], mc, mf, ro.reshape(-1, 3)[s], rd.reshape(-1, 3)[s], cfg, mode="train",
                                        expressions=expr, background_prior=E.bg[s], latent_code=E.latent)
        loss = torch.nn.functional.mse_loss(out[0], tgt[s]) + torch.nn.functional.mse_loss(out[3], tgt[s])
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    torch.cuda.synchronize()
    assert all(p.grad is None for m in (mc, mf) for p in m.parameters())
    return [("pose", pose.detach().clone()), ("expression", expr.detach().clone()), ("losses", torch.stack(losses))]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("loop", ["training", "fitting"])
def test_dropin_loops_repeat_under_torch_deterministic_mode(E, loop, prec, deterministic, precision):
    """torch.use_deterministic_algorithms(True) is honoured: no op on the path raises, and two runs of the same 10-step loop end
    with equal parameters (latent codes, or expression and pose).  torch also fills uninitialised outputs (torch.empty) with
    NaN in this mode, so a gradient element the library failed to write would show up."""
    precision(prec)
    fr = O.synthetic_frame(21, 48, 48)
    idx, tgt = _batches(E, 10, 43)
    run = _reference_style_training if loop == "training" else _fitting
    a, b = run(E, 10, idx, tgt, fr), run(E, 10, idx, tgt, fr)
    _assert_equal(a, b, f"{loop} {prec}")
