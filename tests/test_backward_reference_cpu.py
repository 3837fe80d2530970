"""Pins the floating-point reference of the fused backward kernels (tests/torch_reference.py: render_at_depths, what
tests/test_backward_gpu.py compares the CUDA gradients with) to the UNMODIFIED reference's own autograd: the training loss of
train_transformed_rays.py:355-389 (mse of the coarse and the fine colour against the target) is back-propagated through the live
reference's run_one_iter_of_nerf (mode "train", perturbation and sigma noise on, background image) and through render_at_depths at
the depths the reference sampled; parameter gradients of both networks and the latent-code gradient must agree to FP32 rounding.

So the chain for SURVEY.md §8 row a11 is: CUDA backward  <->  torch_reference (GPU tests)  <->  reference autograd (this file).
What the reference computed (its outputs, its four random draws, the loss, the latent gradient and a fixed sample of 512
entries plus the max |g| of every parameter gradient) was recorded by running it (oracle/make_golden_live.py ->
tests/golden/live/backward.npz); CPU only."""
import os

import pytest
import torch

import golden_io
import make_golden_live as ML
import nerface_oracle as O
import torch_reference as TR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "backward.npz")
# float64 reference vs the stored FP32 autograd gradients, relative to each tensor's max: measured 5.6e-6 (random init),
# 1.7e-4 (opaque stress, fine layers_dir.0.bias: a sum over every sample in which the FP32 autograd's own accumulation error
# shows).  20x below the 1e-2 the GPU tests allow the kernels.
FP64_TOL = 5e-4


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(GOLD)


@pytest.mark.parametrize("stress,white,use_bg", [(False, False, True), (True, False, True), (True, True, False)],
                         ids=["random_init", "opaque_stress", "opaque_stress_white_nobg"])
def test_torch_reference_gradients_equal_reference_autograd(gold, stress, white, use_bg, request):
    tag = request.node.callspec.id
    g = gold[tag]
    H, W, s, fr, pc, pf, ro, rd, bg, target = ML.backward_inputs(stress, white, use_bg)
    near, far = ML.NEAR, ML.FAR
    out = g["out"]
    draws = g["draws"]
    assert len(draws) == 4  # rand[N,Nc], randn[N,Nc], rand[N,Nf], randn[N,Nc+Nf] (train_utils.py:69-76, 105-119)
    noise = O.Noise(t_rand=draws[0], n_c=draws[1], u=draws[2], n_f=draws[3])

    # ---- the depths the reference sampled (the oracle reproduces the forward bit for bit, test_oracle_vs_reference_cpu.py)
    rays = torch.cat((ro, rd, near * torch.ones_like(rd[:, :1]), far * torch.ones_like(rd[:, :1])), dim=-1)
    ex = {}
    with torch.no_grad():
        o_out = O.render_chunk(rays, pc, pf, s, fr["expr"], fr["latent"], bg, noise, extras=ex)
    for a, b in zip(out, o_out):
        assert torch.equal(a, b)

    # ---- the backward tests' floating-point reference at those depths
    lc = {k: v.clone().requires_grad_(True) for k, v in pc.items()}
    lf = {k: v.clone().requires_grad_(True) for k, v in pf.items()}
    lat = fr["latent"].clone().requires_grad_(True)
    got = TR.render_at_depths(rays, lc, lf, fr["expr"], lat, ex["z_coarse"], ex["z_fine"], near, far, 0.1,
                              {"n_c": noise.n_c, "n_f": noise.n_f}, white, bg, None)
    for i in (0, 1, 2, 3, 4, 5, 6):
        assert float((got[i].detach() - out[i]).abs().max()) <= 2e-6 * max(1.0, float(out[i].abs().max())), i
    loss = torch.nn.functional.mse_loss(got[0], target) + torch.nn.functional.mse_loss(got[3], target)
    assert abs(float(loss.detach()) - g["loss"]) <= 1e-7
    loss.backward()

    def close(a, b, scale, what):
        scale = max(scale, 1e-12)
        assert float((a - b).abs().max()) <= 2e-5 * scale, (what, float((a - b).abs().max()), scale)

    n_checked = 0
    for leaves, tag_net in ((lc, "coarse"), (lf, "fine")):
        for k in TR.PARAM_ORDER:
            ref = g["grads"][f"{tag_net}/{k}"]
            if k.startswith("layers_dir.3"):  # built by the reference model but never used by its forward (models.py:257)
                assert ref is None and leaves[k].grad is None
                continue
            assert ref is not None and leaves[k].grad is not None, (tag_net, k)
            ours = leaves[k].grad
            assert list(ours.shape) == ref["shape"]
            close(ours.reshape(-1)[torch.from_numpy(ref["index"])], ref["value"], ref["absmax"], (tag_net, k))
            assert abs(float(ours.abs().max()) - ref["absmax"]) <= 2e-5 * max(ref["absmax"], 1e-12), (tag_net, k)
            n_checked += 1
    assert n_checked == 2 * 24
    close(lat.grad, g["latent_grad"], float(g["latent_grad"].abs().max()), "latent")
    assert float(g["latent_grad"].abs().max()) > 0


@pytest.mark.parametrize("stress,white,use_bg", [(False, False, True), (True, False, True), (True, True, False)],
                         ids=["random_init", "opaque_stress", "opaque_stress_white_nobg"])
def test_torch_reference_in_float64_matches_reference_autograd(gold, stress, white, use_bg, request):
    """tests/test_backward_fp64_gpu.py evaluates render_at_depths in float64: with every input cast to float64 (at the FP32
    depths the reference sampled) it must stay dtype-clean and agree with the reference's FP32 autograd to within FP32
    accumulation error (FP64_TOL)."""
    g = gold[request.node.callspec.id]
    H, W, s, fr, pc, pf, ro, rd, bg, target = ML.backward_inputs(stress, white, use_bg)
    near, far = ML.NEAR, ML.FAR
    draws = g["draws"]
    noise = O.Noise(t_rand=draws[0], n_c=draws[1], u=draws[2], n_f=draws[3])
    rays = torch.cat((ro, rd, near * torch.ones_like(rd[:, :1]), far * torch.ones_like(rd[:, :1])), dim=-1)
    ex = {}
    with torch.no_grad():
        O.render_chunk(rays, pc, pf, s, fr["expr"], fr["latent"], bg, noise, extras=ex)
    d = torch.float64
    lc = {k: v.to(d).requires_grad_(True) for k, v in pc.items()}
    lf = {k: v.to(d).requires_grad_(True) for k, v in pf.items()}
    lat = fr["latent"].to(d).requires_grad_(True)
    got = TR.render_at_depths(rays.to(d), lc, lf, fr["expr"].to(d), lat, ex["z_coarse"].to(d), ex["z_fine"].to(d), near, far, 0.1,
                              {"n_c": noise.n_c.to(d), "n_f": noise.n_f.to(d)}, white, bg.to(d) if bg is not None else None, None)
    assert all(o.dtype == d for o in got)
    for i in range(7):
        assert float((got[i].detach() - g["out"][i].to(d)).abs().max()) <= 1e-5 * max(1.0, float(g["out"][i].abs().max())), i
    loss = torch.nn.functional.mse_loss(got[0], target.to(d)) + torch.nn.functional.mse_loss(got[3], target.to(d))
    loss.backward()
    worst = (0.0, "")
    for leaves, tag_net in ((lc, "coarse"), (lf, "fine")):
        for k in TR.PARAM_ORDER:
            ref = g["grads"][f"{tag_net}/{k}"]
            if ref is None:
                assert leaves[k].grad is None
                continue
            ours = leaves[k].grad
            assert ours.dtype == d
            scale = max(ref["absmax"], 1e-12)
            e = max(float((ours.reshape(-1)[torch.from_numpy(ref["index"])] - ref["value"].to(d)).abs().max()),
                    abs(float(ours.abs().max()) - ref["absmax"])) / scale
            worst = max(worst, (e, f"{tag_net}/{k}"))
    lg = g["latent_grad"]
    worst = max(worst, (float((lat.grad - lg.to(d)).abs().max()) / float(lg.abs().max()), "latent"))
    print(f"float64 vs the reference's FP32 autograd: worst {worst[0]:.2e} of absmax ({worst[1]})")
    assert worst[0] <= FP64_TOL, worst
