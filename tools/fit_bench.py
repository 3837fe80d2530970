#!/usr/bin/env python
"""Fitting-iteration benchmark: analysis-by-synthesis of one frame with a frozen avatar.  2048 rays of a synthetic 512x512
frame, 64 coarse + 64 fine samples, stratified sampling + sigma noise, expression and camera pose requiring grad, rays from
the pose through get_ray_bundle (torch), loss = mse(rgb_c) + mse(rgb_f), Adam on (expression, pose) — through the drop-in
API (run_one_iter_of_nerf + loss.backward()).

Two backward modes are timed: "input_only" (networks frozen: no parameter gradient is formed, nfb_render_backward_ex's
input-only mode) and "full" (the networks' parameters also require grad, as when the caller trains and fits at once).
Prints one JSON line with the median milliseconds per iteration of each (CUDA events), and for each mode the GPU time per
iteration of every kernel, from torch.profiler over 5 further iterations (<mode>_kernels_us, largest first)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--precision", default="fast")
    a = ap.parse_args()
    import nerface_oracle as O
    import nerf
    from nerf import _engine

    dev = torch.device("cuda", 0)
    _engine.set_precision(a.precision)
    H = W = 512
    fr = O.synthetic_frame(21, H, W)
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=2048)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    models = []
    for seed in (100, 101):
        m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                            include_input_xyz=True, include_input_dir=False)
        m.load_state_dict(O.random_init_params(seed, True))
        models.append(m.to(dev))
    mc, mf = models
    g = torch.Generator().manual_seed(0)
    sel = torch.randperm(H * W, generator=g)[:a.rays].to(dev)
    target = torch.rand(a.rays, 3, generator=g).to(dev)
    lat = fr["latent"].to(dev)
    res = {"metric": "fit_iteration_ms", "rays": a.rays, "samples": "64c+64f", "precision": a.precision,
           "gpu": torch.cuda.get_device_name(0)}

    def kernel_us(prof, iters):
        tot = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                name = e.name.split("(")[0]
                tot[name] = tot.get(name, 0.0) + getattr(e, "device_time", getattr(e, "cuda_time", 0.0)) / iters
        return {k: round(v, 1) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}

    for mode in ("input_only", "full"):
        for m in models:
            m.requires_grad_(mode == "full")
        pose = fr["pose"].to(dev).clone().requires_grad_(True)
        expr = fr["expr"].to(dev).clone().requires_grad_(True)
        opt = torch.optim.Adam([pose, expr], lr=1e-4)
        times = []
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        for it in range(a.warmup + a.steps + 5):
            if it == a.warmup + a.steps:
                prof.start()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            opt.zero_grad(set_to_none=True)
            for m in models:
                m.zero_grad(set_to_none=True)
            ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], pose)
            ro, rd = ro.reshape(-1, 3)[sel], rd.reshape(-1, 3)[sel]
            out = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="train", expressions=expr,
                                            latent_code=lat)
            loss = torch.nn.functional.mse_loss(out[0], target) + torch.nn.functional.mse_loss(out[3], target)
            loss.backward()
            opt.step()
            t1.record()
            torch.cuda.synchronize()
            if a.warmup <= it < a.warmup + a.steps:
                times.append(t0.elapsed_time(t1))
            assert pose.grad is not None and expr.grad is not None
        prof.stop()
        res[f"{mode}_kernels_us"] = kernel_us(prof, 5)
        times.sort()
        res[f"{mode}_ms"] = round(times[len(times) // 2], 3)
        res[f"{mode}_ms_min"] = round(times[0], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
