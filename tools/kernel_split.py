"""Per-kernel GPU time of fused training steps in each precision mode (torch.profiler, CUDA activity), as tools/train_bench.py
runs them: 2048 rays, 64c+64f, perturbation + noise 0.1, background, Adam.  Prints one JSON line per mode:
{"precision", "steps", "kernels": {name: ms per step}, "total_ms": ms per step}.

    python tools/kernel_split.py [--steps 10] [--precision fast exact exact_grad]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--precision", nargs="+", default=["fast", "exact", "exact_grad"])
    a = ap.parse_args()
    import nerf
    import nerface_oracle as O
    from nerf import fused_train
    dev = torch.device("cuda", 0)
    H = W = 512
    fr = O.synthetic_frame(0, H, W)
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(dev))
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    bg = fr["bg"].reshape(-1, 3).to(dev)
    target = torch.rand(H * W, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    expr = fr["expr"].to(dev)
    for prec in a.precision:
        mk = lambda seed: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
            num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
        mc, mf = mk(0), mk(1)
        mc.load_state_dict(O.random_init_params(100))
        mf.load_state_dict(O.random_init_params(101))
        mc, mf = mc.to(dev), mf.to(dev)
        t = fused_train.FusedTrainer(mc, mf, n_latent=16, lr=5e-4, num_coarse=64, num_fine=64, perturb=True, noise_std=0.1, near=0.2,
                                     far=0.8, latent_reg=0.005, precision=prec)
        g = torch.Generator(device=dev).manual_seed(7)
        idx = [torch.randint(0, H * W, (a.rays,), device=dev, generator=g) for _ in range(a.steps + 2)]

        def step(i):
            sel = idx[i]
            t.gradients(ro[sel], rd[sel], target[sel], expr, 3, background=bg[sel])
            t.update()

        for i in range(2):
            step(i)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(a.steps):
                step(2 + i)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                per[e.key] = per.get(e.key, 0.0) + us / 1000.0 / a.steps
        top = dict(sorted(per.items(), key=lambda kv: -kv[1])[:14])
        print(json.dumps({"precision": prec, "steps": a.steps, "total_ms": round(sum(per.values()), 3),
                          "kernels": {k[:60]: round(v, 3) for k, v in top.items()}}))


if __name__ == "__main__":
    main()
