"""Parity where round 1 was thin (VERDICT r1, "Harden parity"): the FULL problem sizes of BASELINE.json's configurations against
the oracle (rays sampled across every CTA and every iteration of the persistent kernel), the fast mode's accuracy on
trained-like (opaque) weights as a PSNR gate, the chunk-level entry predict_and_render_radiance, the per-layer activation
probe, and stochastic evaluation (the shipped YAML's validation block has perturb: True)."""
import math
import os

import numpy as np
import pytest
import torch

import nerface_oracle as O

pytestmark = pytest.mark.gpu
NAMES = ["rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last"]
GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")


def make_model(nerf, params, dev):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params)
    return m.to(dev)


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine
    return nerf, _engine, torch.device("cuda", 0)


def psnr(a, b):
    mse = float(((a - b) ** 2).mean())
    return 99.0 if mse == 0 else -10.0 * math.log10(mse)


@pytest.mark.parametrize("H,nc,nf,n_samp", [(512, 64, 128, 4096), (1024, 128, 256, 4096)], ids=["512_64c128f", "1024_128c256f"])
def test_full_frame_against_oracle(env, H, nc, nf, n_samp):
    """BASELINE configs 2 and 4 at FULL size: the whole frame is rendered in one launch (every SM's CTA, hundreds of units each),
    4096 rays spread evenly over the launch — every CTA, early and late iterations, all four ray slots of a unit — are compared
    with the oracle in both precision modes (north_star: 1e-4 max-abs on random-init weights)."""
    nerf, _engine, dev = env
    W = H
    fr = O.synthetic_frame(1, H, W)
    pc, pf = O.random_init_params(100), O.random_init_params(101)
    eng = _engine.renderer_for(dev)
    eng.sync_weights(make_model(nerf, pc, dev), make_model(nerf, pf, dev))
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    bg = fr["bg"].reshape(-1, 3)
    n = H * W
    k = torch.arange(n_samp)
    pick = (k * (n // n_samp) + (k % 4) + 4 * ((k // 4) % 37)).clamp(max=n - 1)  # consecutive picks land in different units / CTAs
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    rays = torch.cat((ro.reshape(-1, 3)[pick], rd.reshape(-1, 3)[pick], torch.full((n_samp, 1), 0.2), torch.full((n_samp, 1), 0.8)), dim=-1)
    with torch.no_grad():
        ref = O.render_chunk(rays, pc, pf, O.Sampling(nc, nf, False, 0.0, False, 65536), fr["expr"], fr["latent"], bg[pick], O.Noise())
    for prec in ("fast", "exact"):
        v = eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, 0.2, 0.8, nc, nf, background=bg.to(dev).contiguous(), precision=prec)
        torch.cuda.synchronize()
        errs = {name: float((v[name].cpu()[pick].reshape(r.shape) - r).abs().max()) for name, r in zip(NAMES, ref)}
        print(f"{H}x{W} {nc}c+{nf}f {prec}: " + " ".join(f"{a}={b:.2e}" for a, b in errs.items()))
        assert max(errs.values()) < 1e-4, (prec, errs)
        assert torch.isfinite(v["_buf"]).all()


@pytest.mark.parametrize("case", ["det_stress_64c128f", "stoch_stress_chunks"])
def test_fast_mode_psnr_on_opaque_stress(env, case):
    """SURVEY.md §8d: fast mode (single FP16 operands) is gated by PSNR against the reference's outputs on the opaque-stress
    weights, where FP16 operand error is not hidden by transparency.  Measured: rgb 79.9 dB (max-abs 1.4e-3), disp max-abs
    1.6e-2 on values of 1..5 (512x512 rows); 82.2 dB / 71.9 dB on the two golden cases; gates: rgb_fine >= 68 dB, rgb max-abs <= 4e-3,
    disp max-abs <= 4e-2.  Exact mode on the same
    case stays within 3e-4 / 2e-3 (test_render_gpu.py)."""
    nerf, _engine, dev = env
    g = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    T = lambda k: torch.from_numpy(g[k]).to(dev) if k in g.files else None  # noqa: E731
    pc, pf = O.random_init_params(int(g["seed_coarse"]), True), O.random_init_params(int(g["seed_fine"]), True)
    eng = _engine.renderer_for(dev)
    eng.sync_weights(make_model(nerf, pc, dev), make_model(nerf, pf, dev))
    eng.set_frame(T("expr"), T("latent"))
    noise = {k: T("noise_" + k) for k in ("t_rand", "n_c", "u", "n_f")}
    out = eng.render(T("ro").reshape(-1, 3), T("rd").reshape(-1, 3), float(g["near"]), float(g["far"]), int(g["num_coarse"]),
                     int(g["num_fine"]), perturb=bool(g["perturb"]), noise_std=float(g["noise_std"]), background=T("bg"),
                     noise=noise if any(v is not None for v in noise.values()) else None, precision="fast")
    torch.cuda.synchronize()
    ref_rgb, ref_disp = torch.from_numpy(g["out3"]).reshape(-1, 3), torch.from_numpy(g["out4"]).reshape(-1)
    got_rgb, got_disp = out["rgb_fine"].cpu(), out["disp_fine"].cpu()
    p = psnr(got_rgb, ref_rgb)
    print(f"{case} fast: rgb_fine PSNR {p:.1f} dB, max|d rgb| {float((got_rgb - ref_rgb).abs().max()):.2e}, "
          f"max|d disp| {float((got_disp - ref_disp).abs().max()):.2e}; min w_last {float(torch.from_numpy(g['out6']).min()):.3f}")
    assert p >= 68.0
    assert float((got_rgb - ref_rgb).abs().max()) <= 4e-3 and float((got_disp - ref_disp).abs().max()) <= 4e-2
    assert float(torch.from_numpy(g["out6"]).min()) < 0.1  # the case really is opaque somewhere


def _cfg(nerf, **over):
    blk = dict(num_coarse=64, num_fine=128, perturb=False, lindisp=False, radiance_field_noise_std=0.0, white_background=False, chunksize=16)
    blk.update(over)
    return nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, validation=blk, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_predict_and_render_radiance_direct(env, precision):
    """The chunk-level entry (train_utils.py:36-162) called the way the reference's driver calls it: a [N, 8] ray batch, with
    and without the ablation bundle `ray_dirs_fake` (a list of chunks; chunk 0's column 5 feeds the direction encoder, :81-82)."""
    nerf, _engine, dev = env
    nerf.set_precision(precision)
    try:
        n = 16
        fr = O.synthetic_frame(8, 4, 4)
        pc, pf = O.random_init_params(100), O.random_init_params(101)
        mc, mf = make_model(nerf, pc, dev), make_model(nerf, pf, dev)
        ro, rd = O.ray_bundle(4, 4, fr["intrinsics"], fr["pose"])
        rays = torch.cat((ro.reshape(-1, 3), rd.reshape(-1, 3), torch.full((n, 1), 0.2), torch.full((n, 1), 0.8)), dim=-1)
        bg = fr["bg"].reshape(-1, 3)
        kw = dict(expressions=fr["expr"].to(dev), background_prior=bg.to(dev), latent_code=fr["latent"].to(dev))
        cfg = _cfg(nerf)
        with torch.no_grad():
            got = nerf.predict_and_render_radiance(rays.to(dev), mc, mf, cfg, mode="validation", **kw)
            ref = O.render_chunk(rays, pc, pf, O.Sampling(64, 128), fr["expr"], fr["latent"], bg, O.Noise())
        assert len(got) == 7
        for name, a, b in zip(NAMES, got, ref):
            assert a.shape == b.shape and float((a.cpu() - b).abs().max()) < 1e-4, name
        fr2 = O.synthetic_frame(9, 4, 4)
        _, rd2 = O.ray_bundle(4, 4, fr2["intrinsics"], fr2["pose"])
        fake = torch.cat((ro.reshape(-1, 3), rd2.reshape(-1, 3), torch.full((n, 1), 0.2), torch.full((n, 1), 0.8)), dim=-1)
        with torch.no_grad():
            got = nerf.predict_and_render_radiance(rays.to(dev), mc, mf, cfg, mode="validation", ray_dirs_fake=[fake.to(dev)], **kw)
            dir_cols = torch.cat((fake[:, 5:6], rays[:, 6:8]), dim=-1)
            ref = O.render_chunk(rays, pc, pf, O.Sampling(64, 128), fr["expr"], fr["latent"], bg, O.Noise(), dir_cols=dir_cols)
        for name, a, b in zip(NAMES, got, ref):
            assert float((a.cpu() - b).abs().max()) < 1e-4, name
        assert float((got[3].cpu() - nerf.predict_and_render_radiance(rays.to(dev), mc, mf, cfg, mode="validation", **kw)[3].cpu()).abs().max()) > 1e-6
    finally:
        nerf.set_precision("fast")


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_layer_probe_against_oracle_activations(env, precision):
    """NfbDebug.act_step: the post-activation values the epilogue of every tensor-core step produced for the first 128 coarse
    rows, against the oracle's layer outputs (models.py:244-257 order: six layers_xyz, three layers_dir) — localises an error
    to a layer, which the end-to-end outputs cannot.  Exact: 2e-5; fast: FP16 operands, 2e-3 of the layer's largest value."""
    nerf, _engine, dev = env
    fr = O.synthetic_frame(12, 2, 2)
    pc = O.random_init_params(100, True)
    mc, mf = make_model(nerf, pc, dev), make_model(nerf, O.random_init_params(101, True), dev)
    eng = _engine.renderer_for(dev)
    eng.sync_weights(mc, mf)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    ro, rd = O.ray_bundle(2, 2, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    z = 0.2 * (1.0 - torch.linspace(0.0, 1.0, 64)) + 0.8 * torch.linspace(0.0, 1.0, 64)
    pts = (ro[:2, None, :] + rd[:2, None, :] * z[None, :, None])          # rays 0, 1 = the first 128 coarse rows
    dirs = torch.cat((rd[:2, 2:3], torch.full((2, 1), 0.2), torch.full((2, 1), 0.8)), dim=-1)
    x = O._encode(pts, dirs)
    acts = O.mlp_activations(pc, x, fr["expr"], fr["latent"])
    tol = 2e-5 if precision == "exact" else 2e-3
    for step, ref in enumerate(acts):
        out = eng.render(ro.to(dev), rd.to(dev), 0.2, 0.8, 64, 128, background=fr["bg"].reshape(-1, 3).to(dev), precision=precision,
                         act_step=step)
        torch.cuda.synchronize()
        got = out["act"].cpu()[:, :ref.shape[1]]
        scale = max(1.0, float(ref.abs().max())) if precision == "fast" else 1.0
        err = float((got - ref).abs().max())
        assert err <= tol * scale, (step, err, float(ref.abs().max()))


def test_stochastic_evaluation_like_the_shipped_yaml(env):
    """…paper_model.yml:158 evaluates with perturb: True, i.e. stochastically: the seeded drop-in call must equal the oracle
    fed with the same draws (the reference's per-chunk draw order), through the pipelined kernel."""
    nerf, _engine, dev = env
    H, W = 6, 8
    fr = O.synthetic_frame(13, H, W)
    pc, pf = O.random_init_params(100), O.random_init_params(101)
    mc, mf = make_model(nerf, pc, dev), make_model(nerf, pf, dev)
    cfg = _cfg(nerf, perturb=True, num_fine=64, chunksize=65536)
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(dev))
    kw = dict(expressions=fr["expr"].to(dev), background_prior=fr["bg"].reshape(-1, 3).to(dev), latent_code=fr["latent"].to(dev))
    torch.manual_seed(5)
    with torch.no_grad():
        got = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="validation", **kw)
    torch.manual_seed(5)
    n = H * W
    noise = O.Noise(t_rand=torch.rand((n, 64), device=dev).cpu(), u=torch.rand((n, 64), device=dev).cpu())
    cro, crd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    with torch.no_grad():
        ref = O.run_one_iter(cro, crd, pc, pf, O.Sampling(64, 64, True, 0.0, False, 65536), 0.2, 0.8, fr["expr"], fr["latent"],
                             fr["bg"].reshape(-1, 3), "validation", noise_per_chunk=[noise])
    for name, a, b in zip(NAMES, got, ref):
        assert a.shape == b.shape and float((a.cpu() - b).abs().max()) < 1e-4, name
    with torch.no_grad():
        again = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="validation", **kw)
    assert float((again[3] - got[3]).abs().max()) > 0  # a second call draws fresh samples


@pytest.mark.parametrize("n", [1, 2, 3, 5, 9])
def test_tiny_ray_counts_through_the_pipelined_kernel(env, n):
    """Fewer rays than one unit of work / than one cluster of CTAs: partly valid units, idle CTAs, a single pipeline block."""
    nerf, _engine, dev = env
    fr = O.synthetic_frame(17, 4, 4)
    ro, rd = O.ray_bundle(4, 4, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3)[:n].contiguous(), rd.reshape(-1, 3)[:n].contiguous()
    bg = fr["bg"].reshape(-1, 3)[:n].contiguous()
    pc, pf = O.random_init_params(100, True), O.random_init_params(101, True)
    eng = _engine.renderer_for(dev)
    eng.sync_weights(make_model(nerf, pc, dev), make_model(nerf, pf, dev))
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    rays = torch.cat((ro, rd, torch.full((n, 1), 0.2), torch.full((n, 1), 0.8)), dim=-1)
    with torch.no_grad():
        ref = O.render_chunk(rays, pc, pf, O.Sampling(64, 128), fr["expr"], fr["latent"], bg, O.Noise())
    out = eng.render(ro.to(dev), rd.to(dev), 0.2, 0.8, 64, 128, background=bg.to(dev), precision="fast")
    torch.cuda.synchronize()
    for name, r in zip(NAMES, ref):
        tol = 4e-2 if name.startswith("disp") else 4e-3  # opaque-stress weights, fast mode (see test_render_gpu.tolerance)
        assert float((out[name].cpu() - r).abs().max()) <= tol, (n, name)
