"""Pins the floating-point reference of the input gradients (tests/torch_reference.render_at_depths with the rays, expression,
background and dir_z as leaves: what tests/test_input_grads_gpu.py compares the CUDA input gradients with) to the UNMODIFIED
reference's own autograd.

The reference's run_one_iter_of_nerf (mode "train", perturbation and sigma noise on) was back-propagated from the training loss
with ray_origins, ray_directions, expressions, background_prior and latent_code requiring grad, and in the "ablation" case also
ray_directions_ablation, over two chunks whose direction encoder both read chunk 0 of the ablation bundle
(oracle/make_golden_inputs.py -> tests/golden/live/backward_inputs.npz).  Here the same loss goes through render_at_depths at the
depths the reference sampled; dir_z is built from the ablation leaf by the drop-in's own slicing (nerf/train_utils.py), so the
ablation gradient checks that routing too.  Compared per tensor, relative to its max |g|: FP32 within 2e-5, float64 within 5e-4
(the float64 bound of test_backward_reference_cpu.py).  CPU only."""
import os

import pytest
import torch

import golden_io
import make_golden_inputs as MI
import make_golden_live as ML
import nerface_oracle as O
import torch_reference as TR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "backward_inputs.npz")
FP32_TOL = 2e-5  # measured worst 4.2e-7 (ablation case, latent_code)
FP64_TOL = 5e-4  # measured worst 1.1e-4 (opaque_stress_white_nobg, ray_directions)


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(GOLD)


def _noise(draws):
    """The reference draws four tensors per chunk (train_utils.py:69-76, 105-119): concatenate them per kind."""
    assert len(draws) % 4 == 0
    return O.Noise(*[torch.cat(draws[k::4], dim=0) for k in range(4)])


def _run(g, tag, dtype):
    stress, white, use_bg, ablation, chunk = MI.INPUT_CASES[tag]
    H, W, s, fr, pc, pf, ro, rd, bg, target = ML.backward_inputs(stress, white, use_bg)
    near, far = ML.NEAR, ML.FAR
    inp = g["inputs"]
    assert torch.equal(inp["ray_origins"], ro) and torch.equal(inp["ray_directions"], rd)
    noise = _noise(g["draws"])
    n = ro.shape[0]
    abl = inp.get("ray_directions_ablation")
    dir_z = None
    if abl is not None:  # every chunk sees chunk 0 of the ablation bundle (train_utils.py:81-82)
        dir_z = torch.cat([abl[:chunk, 2]] * ((n + chunk - 1) // chunk))[:n]
    rays = torch.cat((ro, rd, near * torch.ones_like(rd[:, :1]), far * torch.ones_like(rd[:, :1])), dim=-1)
    ex = {}
    dir_cols = torch.stack((dir_z, rays[:, 6], rays[:, 7]), -1) if dir_z is not None else None
    with torch.no_grad():
        o_out = O.render_chunk(rays, pc, pf, s, fr["expr"], fr["latent"], bg, noise, dir_cols=dir_cols, extras=ex)
    for a, b in zip(g["out"], o_out):  # the oracle reproduces the reference's forward, so these are its depths
        assert torch.equal(a, b)

    leaf = lambda t: t.detach().to(dtype).clone().requires_grad_(True)  # noqa: E731
    L = {k: leaf(v) for k, v in inp.items()}
    rays = torch.cat((L["ray_origins"], L["ray_directions"], torch.full((n, 2), 0.0, dtype=dtype) + torch.tensor([near, far], dtype=dtype)), -1)
    dz = None
    if abl is not None:
        dz = torch.cat([L["ray_directions_ablation"][:chunk, 2]] * ((n + chunk - 1) // chunk))[:n]
    got = TR.render_at_depths(rays, {k: v.to(dtype) for k, v in pc.items()}, {k: v.to(dtype) for k, v in pf.items()},
                              L["expressions"], L["latent_code"], ex["z_coarse"].to(dtype), ex["z_fine"].to(dtype), near, far, 0.1,
                              {"n_c": noise.n_c.to(dtype), "n_f": noise.n_f.to(dtype)}, white, L.get("background_prior"), dz)
    for i in range(7):
        assert float((got[i].detach() - g["out"][i].to(dtype)).abs().max()) <= 1e-5 * max(1.0, float(g["out"][i].abs().max())), i
    loss = torch.nn.functional.mse_loss(got[0], target.to(dtype)) + torch.nn.functional.mse_loss(got[3], target.to(dtype))
    loss.backward()
    worst = (0.0, "")
    for k, ref in g["grads"].items():
        ours = L[k].grad
        assert ours is not None and ours.dtype == dtype and ours.shape == ref.shape, k
        scale = float(ref.abs().max())
        assert scale > 0, k
        worst = max(worst, (float((ours - ref.to(dtype)).abs().max()) / scale, k))
    print(f"{tag} {dtype}: worst {worst[0]:.2e} of absmax ({worst[1]})")
    return worst, set(g["grads"])


CASES = list(MI.INPUT_CASES)


@pytest.mark.parametrize("tag", CASES)
def test_input_gradients_fp32_equal_reference_autograd(gold, tag):
    worst, names = _run(gold[tag], tag, torch.float32)
    assert {"ray_origins", "ray_directions", "expressions", "latent_code"} <= names
    assert worst[0] <= FP32_TOL, worst


@pytest.mark.parametrize("tag", CASES)
def test_input_gradients_float64_match_reference_autograd(gold, tag):
    worst, names = _run(gold[tag], tag, torch.float64)
    if tag == "ablation":
        assert "ray_directions_ablation" in names
    assert worst[0] <= FP64_TOL, worst


def test_ablation_gradient_reaches_chunk_zero_only(gold):
    """The reference's ablation directions receive gradient only in chunk 0's z column (what every chunk's encoder read)."""
    g = gold["ablation"]["grads"]["ray_directions_ablation"]
    chunk = MI.INPUT_CASES["ablation"][4]
    assert float(g[:chunk, 2].abs().max()) > 0
    assert float(g[chunk:].abs().max()) == 0.0 and float(g[:, :2].abs().max()) == 0.0
