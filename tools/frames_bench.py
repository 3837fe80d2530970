#!/usr/bin/env python
"""Multi-frame benchmark (nfb_set_frames / nfb_render_*_frames*): what conditioning every ray on its own frame costs.

  eval : the rays of one synthetic 512x512 frame, 64 coarse + 128 fine samples, fast mode, rendered (a) with the single-frame
         kernel after nfb_set_frame, (b) as ONE multi-frame call over F = 8 frames, frame index = ray % 8 (every unit and tile
         mixes frames).  Same rays, same sample counts; rays/s of each.
  fit  : one fitting iteration of 8 frames x 256 rays, 64c + 64f, stratified sampling + sigma noise, a frozen avatar
         (input-only backward: per-frame expression and latent gradients), (a) as 8 single-frame iterations (set_frame, training
         forward, backward each), (b) as one joint multi-frame iteration; and the same with parameter gradients ("train").

Timings are CUDA-event medians over --steps repetitions after --warmup, with the min and max beside them.  Prints one JSON line."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return dict(median_ms=ms[len(ms) // 2], min_ms=ms[0], max_ms=ms[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    a = ap.parse_args()
    import nerface_oracle as O
    import nerf
    from nerf import _engine

    dev = torch.device("cuda", 0)
    fr = O.synthetic_frame(21, 512, 512)
    ro, rd = O.ray_bundle(512, 512, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3).to(dev).contiguous(), rd.reshape(-1, 3).to(dev).contiguous()
    models = []
    for seed in (100, 101):
        m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                            include_input_xyz=True, include_input_dir=False)
        m.load_state_dict(O.random_init_params(seed, False))
        models.append(m.to(dev))
    mc, mf = models
    eng = _engine.renderer_for(dev)
    eng.sync_weights(mc, mf)
    F = a.frames
    g = torch.Generator().manual_seed(0)
    ex = (fr["expr"].reshape(1, 76) + 0.3 * torch.randn(F, 76, generator=g)).to(dev).contiguous()
    la = (fr["latent"].reshape(1, 32) + 0.3 * torch.randn(F, 32, generator=g)).to(dev).contiguous()
    res = {"metric": "multi_frame", "gpu": torch.cuda.get_device_name(0), "frames": F, "steps": a.steps}

    # ---- evaluation, one 512x512 frame's rays
    n = ro.shape[0]
    fi = (torch.arange(n, device=dev) % F).to(torch.int32)
    eng.set_frame(ex[0], la[0])
    eng.set_frames(ex, la)
    ev = dict(rays=n, samples="64c+128f", precision="fast")
    for name, kw in (("single_frame", {}), ("multi_frame", dict(frame_index=fi))):
        t = timed(lambda: eng.render(ro, rd, 0.2, 0.8, 64, 128, precision="fast", **kw), a.steps, a.warmup)
        t["rays_per_s"] = n / (t["median_ms"] * 1e-3)
        ev[name] = t
    ev["multi_over_single_time"] = ev["multi_frame"]["median_ms"] / ev["single_frame"]["median_ms"]
    res["eval"] = ev

    # ---- fitting iteration: 8 frames x 256 rays
    per = 256
    sel = torch.randperm(n, generator=g)[:F * per].to(dev)
    fro, frd = ro[sel].contiguous(), rd[sel].contiguous()
    ffi = torch.arange(F, device=dev, dtype=torch.int32).repeat_interleave(per)  # frame f = rays [256 f, 256 f + 256)
    noise = dict(t_rand=torch.rand(F * per, 64, device=dev), n_c=torch.randn(F * per, 64, device=dev),
                 u=torch.rand(F * per, 64, device=dev), n_f=torch.randn(F * per, 128, device=dev))
    pc = eng._params(mc)
    pf = eng._params(mf)
    args = dict(perturb=True, noise_std=0.1, precision="fast", train=True)

    def gouts(out):
        return [torch.ones_like(out["rgb_coarse"]), None, None, torch.ones_like(out["rgb_fine"]), None, None, None]

    def single(want_params):
        def run():
            for f in range(F):
                s = slice(f * per, (f + 1) * per)
                eng.set_frame(ex[f], la[f])
                out = eng.render(fro[s], frd[s], 0.2, 0.8, 64, 64, noise={k: v[s] for k, v in noise.items()}, **args)
                eng.backward(gouts(out), pc, pf, want_params=want_params, inputs=["expression"])
        return run

    def joint(want_params):
        def run():
            eng.set_frames(ex, la)
            out = eng.render(fro, frd, 0.2, 0.8, 64, 64, noise=noise, frame_index=ffi, **args)
            eng.backward(gouts(out), pc, pf, want_params=want_params, inputs=["expression"], frames=True)
        return run

    fit = dict(rays=F * per, samples="64c+64f", precision="fast")
    for mode, wp in (("input_only", False), ("train", True)):
        s, j = timed(single(wp), a.steps, a.warmup), timed(joint(wp), a.steps, a.warmup)
        fit[mode] = dict(single_frame_x8=s, joint=j, joint_over_single=j["median_ms"] / s["median_ms"])
    res["fit"] = fit
    print(json.dumps(res))


if __name__ == "__main__":
    main()
