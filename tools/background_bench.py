#!/usr/bin/env python
"""What learning the background costs in the fused K-image training step (DESIGN.md 8e): 512x512 synthetic frames, 64 coarse +
64 fine samples, stratified sampling + sigma noise 0.1, 2048 rays per step in all, FusedTrainer.step_images_graph at K = 1 and
K = 8 in three configurations, alternated in one process:

  * fixed      — the training set's own background (TrainImages(background=...)), as before;
  * learned    — FusedTrainer(background=mean image): the bucket's background rows, their gradient rows, Adam over them;
  * supervised — learned + background_loss=0.001 (the reference's supervised_train_background term).

Per configuration: --warmup steps, then --steps steps between two CUDA events, --rounds times in turn; the median ms per
step is reported, with every round's value.  Prints one JSON line with the card's name and power limit read in the same
process, the library launches per eager step, and the gradient bucket's size."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001  (no nvidia-smi: the number is reported without it)
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--rays", type=int, default=2048)
    a = ap.parse_args()
    import nerface_oracle as O
    import nerf
    from nerf import _engine, fused_train, ray_sampler

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    H = W = 512
    n_img = a.images
    frs = [O.synthetic_frame(i, H, W) for i in range(n_img)]
    images = torch.rand(n_img, H, W, 3, generator=torch.Generator().manual_seed(1)).to(dev)
    bboxs = [(150 + 4 * i, 400, 128, 380 - 3 * i) for i in range(n_img)]
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs]).to(dev)
    fixed = ray_sampler.TrainImages(images, poses, exprs, bboxs, frs[0]["intrinsics"], background=frs[0]["bg"].to(dev), device=dev)
    plain = ray_sampler.TrainImages(images, poses, exprs, bboxs, frs[0]["intrinsics"], device=dev)
    eng = _engine.renderer_for(dev)
    init = images.mean(0)  # the reference's initialisation of a learned background

    def trainer(**kw):
        mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
            num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
        mc, mf = mk(), mk()
        mc.load_state_dict(O.random_init_params(100))
        mf.load_state_dict(O.random_init_params(101))
        return fused_train.FusedTrainer(mc.to(dev), mf.to(dev), n_latent=n_img, num_coarse=64, num_fine=64, perturb=True,
                                        noise_std=0.1, **kw)

    kinds = dict(fixed=(fixed, {}), learned=(plain, dict(background=init)), supervised=(plain, dict(background=init, background_loss=0.001)))
    rng = torch.Generator().manual_seed(2)
    configs, launches, floats = {}, {}, {}
    built = []
    for k in (8, 1):  # the larger step first: it sizes the renderer's buffers every graph then shares
        for kind, (data, kw) in kinds.items():
            t = trainer(**kw)
            n = a.rays // k
            t.step_images(data, list(range(k)), n)
            l0 = eng.launch_count()
            t.step_images(data, list(range(k)), n)
            launches[f"{kind} K={k}"] = eng.launch_count() - l0
            floats[kind] = t.params.numel()
            built.append((f"{kind} K={k}", t, data, k, n))
    for name, t, data, k, n in built:
        t.capture_images(data, k, n)
        idx = torch.empty(k, dtype=torch.int32).pin_memory()
        configs[name] = (lambda t=t, k=k, idx=idx: (idx.copy_(torch.randint(n_img, (k,), generator=rng, dtype=torch.int32)),
                                                         t.step_images_graph(idx)))
    times = {name: [] for name in configs}
    for _ in range(a.rounds):
        for name, fn in configs.items():
            for _ in range(a.warmup):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    res = dict(bench="background_step", card=torch.cuda.get_device_name(dev), power_limit_w=power_limit(), frame=f"{H}x{W}",
               samples="64c+64f", rays_per_step=a.rays, steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               ms_per_step={name: round(statistics.median(v), 3) for name, v in times.items()},
               ms_per_step_all={name: [round(x, 3) for x in v] for name, v in times.items()},
               launches_per_step=launches, bucket_floats=floats)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
