#!/usr/bin/env python
"""SHA-256 digests of everything the library computes on fixed, seeded inputs, for comparing two builds bit for bit (a
refactor of the kernels or of the host layer must leave every digest and the launch count unchanged):

  eval     64c+128f evaluation render of 2304 rays with a background: the seven outputs
  train    2048 rays at 64c+64f, stratified sampling, sigma noise 0.1, background, dir_z: the seven outputs of the training
           forward, all 48 parameter gradients, the latent gradient and the five input gradients
  chunked  the same for 200 rays with NFB_TRAIN_MEM_MB=48 (32 rays per chunk, the last chunk ragged)
  input_only  the train case on other noise with an input-only backward (want_params=False): the seven outputs, the latent
           gradient and the five input gradients, which the PE-only weight-gradient launch serves
  frames   2048 rays of three frames, one multi-frame training forward and backward(frames=True): the seven outputs, the
           parameter gradients, every frame's latent and expression gradient and the other input gradients

each in all three precisions (fast, exact, exact_grad), plus the launches each case took; then, through the host paths above
the renderer:

  dropin/* run_one_iter_of_nerf and render_frames in training mode, then loss.backward(): the outputs and the gradients of
           the parameters, latents, expressions and background
  trainer/*  three steps each of FusedTrainer.step, step_graph, step_images at K = 1 and K = 3, and step_images_graph (K = 3):
           the parameter bucket and the loss after every step

Usage:

  python tools/output_digests.py OUT.json          # NFB_LIB selects the library, as everywhere
  NFB_LIB=/path/to/other/libnfb.so python tools/output_digests.py OTHER.json && cmp OUT.json OTHER.json
"""
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))

NEAR, FAR = 0.2, 0.8
OUTPUTS = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
INPUTS = ["ray_origins", "ray_directions", "expression", "background", "dir_z"]
PRECISIONS = ("fast", "exact", "exact_grad")


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    import nerface_oracle as O
    import nerf
    from nerf import _engine
    from nerf._engine import PARAM_ORDER

    dev = torch.device("cuda", 0)
    eng = _engine.renderer_for(dev)
    fr = O.synthetic_frame(21, 48, 48)
    ro, rd = O.ray_bundle(48, 48, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev)
    bg = fr["bg"].reshape(-1, 3).to(dev)
    expr, latent = fr["expr"].to(dev), fr["latent"].to(dev)

    def model(seed):
        m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
                                                            include_input_dir=False)
        m.load_state_dict(O.random_init_params(seed, True))
        return m.to(dev)

    mc, mf = model(100), model(101)
    pc = [dict(mc.named_parameters())[k] for k in PARAM_ORDER]
    pf = [dict(mf.named_parameters())[k] for k in PARAM_ORDER]
    eng.sync_weights(mc, mf)
    eng.set_frame(expr, latent)
    res = {}

    def record(case, named, l0):
        torch.cuda.synchronize()
        res[case] = {k: digest(t) for k, t in named}
        res[case]["launches"] = eng.launch_count() - l0

    def train_case(case, n, prec, seed, want_params=True):
        g = torch.Generator().manual_seed(seed)
        nz = O.draw_noise(n, O.Sampling(64, 64, True, 0.1, False, 2048), g)
        noise = {k: getattr(nz, k).to(dev) for k in ("t_rand", "n_c", "u", "n_f")}
        dz = (torch.rand(n, generator=g) * 2.0 - 1.0).to(dev)
        shapes = [(n, 3), (n,), (n,), (n, 3), (n,), (n,), (n,)]
        gouts = [((torch.rand(sh, generator=g) - 0.3) / n).to(dev) for sh in shapes]
        l0 = eng.launch_count()
        out = eng.render(ro[:n].contiguous(), rd[:n].contiguous(), NEAR, FAR, 64, 64, perturb=True, noise_std=0.1,
                         background=bg[:n].contiguous(), dir_z=dz, noise=noise, precision=prec, train=True)
        gc, gf, gl, ing = eng.backward(gouts, pc, pf, want_latent=True, want_params=want_params, inputs=INPUTS)
        named = [(k, out[k]) for k in OUTPUTS]
        named += [(f"grad_coarse/{PARAM_ORDER[i]}", t) for i, t in enumerate(gc or []) if t is not None]
        named += [(f"grad_fine/{PARAM_ORDER[i]}", t) for i, t in enumerate(gf or []) if t is not None]
        named += [("grad_latent", gl)] + [("grad_" + k, t) for k, t in sorted(ing.items())]
        record(case, named, l0)

    for prec in PRECISIONS:
        l0 = eng.launch_count()
        out = eng.render(ro, rd, NEAR, FAR, 64, 128, background=bg, precision=prec)
        record(f"eval/{prec}", [(k, out[k]) for k in OUTPUTS], l0)
        train_case(f"train/{prec}", 2048, prec, 1031)
        train_case(f"input_only/{prec}", 2048, prec, 1036, want_params=False)
        os.environ["NFB_TRAIN_MEM_MB"] = "48"  # read by the library on every call
        try:
            train_case(f"chunked/{prec}", 200, prec, 1032)
        finally:
            del os.environ["NFB_TRAIN_MEM_MB"]

    n, nfr = 2048, 3
    g = torch.Generator().manual_seed(1033)
    fexpr, flat = (torch.randn(nfr, 76, generator=g) * 0.5).to(dev), (torch.randn(nfr, 32, generator=g) * 0.1).to(dev)
    fidx = torch.randint(0, nfr, (n,), generator=g).to(dev)
    nz = O.draw_noise(n, O.Sampling(64, 64, True, 0.1, False, 2048), g)
    fnoise = {k: getattr(nz, k).to(dev) for k in ("t_rand", "n_c", "u", "n_f")}
    fdz = (torch.rand(n, generator=g) * 2.0 - 1.0).to(dev)
    fgouts = [((torch.rand(sh, generator=g) - 0.3) / n).to(dev) for sh in [(n, 3), (n,), (n,), (n, 3), (n,), (n,), (n,)]]
    for prec in PRECISIONS:
        l0 = eng.launch_count()
        eng.set_frames(fexpr, flat)
        out = eng.render(ro[:n].contiguous(), rd[:n].contiguous(), NEAR, FAR, 64, 64, perturb=True, noise_std=0.1,
                         background=bg[:n].contiguous(), dir_z=fdz, noise=fnoise, precision=prec, train=True, frame_index=fidx)
        gc, gf, gl, ing = eng.backward(fgouts, pc, pf, want_latent=True, want_params=True, inputs=INPUTS, frames=True)
        named = [(k, out[k]) for k in OUTPUTS]
        named += [(f"grad_coarse/{PARAM_ORDER[i]}", t) for i, t in enumerate(gc) if t is not None]
        named += [(f"grad_fine/{PARAM_ORDER[i]}", t) for i, t in enumerate(gf) if t is not None]
        named += [("grad_latent", gl)] + [("grad_" + k, t) for k, t in sorted(ing.items())]
        record(f"frames/{prec}", named, l0)

    # the drop-in API in training mode: noise drawn by the driver from torch's seeded generator, gradients by loss.backward()
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=1024)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=NEAR, far=FAR)))
    target = torch.rand(n, 3, generator=g).to(dev)
    for case in ("run_one_iter", "render_frames"):
        dc, df = model(100), model(101)
        frames = case == "render_frames"
        e = (fexpr if frames else expr).clone().requires_grad_(True)
        lt = (flat if frames else latent).clone().requires_grad_(True)
        b = bg[:n].clone().requires_grad_(True)
        torch.manual_seed(1034)
        l0 = eng.launch_count()
        if frames:
            outs = nerf.render_frames(ro[:n], rd[:n], fidx, e, lt, dc, df, cfg, background_prior=b)
        else:
            outs = nerf.run_one_iter_of_nerf(48, 48, fr["intrinsics"], dc, df, ro[:n], rd[:n], cfg, mode="train", expressions=e,
                                             background_prior=b, latent_code=lt)
        loss = ((outs[0] - target) ** 2).mean() + ((outs[3] - target) ** 2).mean() + 0.005 * lt.norm()
        loss.backward()
        named = [(k, t) for k, t in zip(OUTPUTS, outs)] + [("loss", loss)]
        named += [(f"grad_coarse/{k}", p.grad) for k, p in dc.named_parameters() if p.grad is not None]
        named += [(f"grad_fine/{k}", p.grad) for k, p in df.named_parameters() if p.grad is not None]
        named += [("grad_latent", lt.grad), ("grad_expression", e.grad), ("grad_background", b.grad)]
        record(f"dropin/{case}", named, l0)

    # FusedTrainer: three steps of each kind from the same initial state, the bucket and the loss after every step
    from nerf import fused_train, ray_sampler
    n_img, H, W, npi = 3, 32, 32, 256
    ifr = [O.synthetic_frame(30 + i, H, W) for i in range(n_img)]
    data = ray_sampler.TrainImages(torch.rand(n_img, H, W, 3, generator=g).to(dev),
                                   torch.stack([f["pose"][:3, :4].reshape(-1) for f in ifr]), torch.stack([f["expr"] for f in ifr]),
                                   [(8, 24, 6, 26), (4, 20, 10, 30), (10, 30, 0, 20)], ifr[0]["intrinsics"],
                                   background=ifr[0]["bg"], device=dev)
    sro, srd, stgt, sbg = ro[:npi].contiguous(), rd[:npi].contiguous(), target[:npi].contiguous(), bg[:npi].contiguous()
    for case in ("step", "step_graph", "step_images_k1", "step_images_k3", "step_images_graph"):
        torch.manual_seed(1035)
        tr = fused_train.FusedTrainer(model(100), model(101), n_latent=n_img, num_coarse=64, num_fine=64, perturb=True,
                                      noise_std=0.1, near=NEAR, far=FAR, latent_codes=torch.randn(n_img, 32, generator=g) * 0.1)
        if case == "step_graph":
            tr.capture(npi)
        elif case == "step_images_graph":
            tr.capture_images(data, 3, npi // 3, max_rounds=8)
        l0 = eng.launch_count()
        named = []
        for i in range(3):
            if case == "step":
                loss = tr.step(sro, srd, stgt, expr, i % n_img, background=sbg)
            elif case == "step_graph":
                loss = tr.step_graph(sro, srd, stgt, expr, i % n_img, background=sbg)
            elif case == "step_images_k1":
                loss = tr.step_images(data, [i % n_img], npi, max_rounds=8)
            elif case == "step_images_k3":
                loss = tr.step_images(data, [i % n_img, (i + 2) % n_img, i % n_img], npi // 3, max_rounds=8)
            else:
                loss = tr.step_images_graph([i % n_img, (i + 2) % n_img, i % n_img])
            named += [(f"params/{i}", tr.params.clone()), (f"loss/{i}", loss.clone())]
        record(f"trainer/{case}", named, l0)

    res["device"] = torch.cuda.get_device_name(0)
    with open(sys.argv[1], "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"{sum(len(v) - 1 for v in res.values() if isinstance(v, dict))} digests -> {sys.argv[1]}")


if __name__ == "__main__":
    main()
