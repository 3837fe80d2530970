#!/usr/bin/env python
"""Training-step benchmark of steps over several images (DESIGN.md 8c): 512x512 synthetic frames, 64 coarse + 64 fine samples,
stratified sampling + sigma noise 0.1, 2048 rays per step in all, alternated in one process:

  * loop   — the single-image loop: RaySampler.sample (host pose, one image) + FusedTrainer.step_graph (copies + replay);
  * K=1..8 — FusedTrainer.step_images_graph: the whole step, sampler included, as one graph replay from K image indices
             (2048 / K rays per image).

Per configuration: --warmup steps, then --steps steps between two CUDA events, --rounds times in turn; the median ms per
step is reported.  Prints one JSON line with the card's name and power limit read in the same process, and the library
launches per step (eager count; a replay issues them from the graph).

--gpus N (N > 1; the script relaunches itself under torch.distributed.run, one rank per GPU, NCCL): the K-image steps run
data-parallel (FusedTrainer.capture_images(world=N)): every rank samples the whole batch and renders 1/N of it, and one
all-reduce of the gradient bucket sits inside each graph.  Besides K = 1..8 at the fixed global batch (strong scaling), the
weak-scaling configuration K = N images x 2048 rays runs, 2048 rays per rank.  Rank 0's CUDA-event times are reported; the
host loop runs at N = 1 only.  The ranks seed torch alike, so their in-graph draws and image indices agree."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist

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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--gpus", type=int, default=1)
    a = ap.parse_args()
    world, rank, local = (int(os.environ.get(v, d)) for v, d in (("WORLD_SIZE", "1"), ("RANK", "0"), ("LOCAL_RANK", "0")))
    if a.gpus > 1 and world == 1:
        if torch.cuda.device_count() < a.gpus:
            sys.exit(f"--gpus {a.gpus}: this machine has {torch.cuda.device_count()} GPU(s)")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={a.gpus}", "--master-addr",
               "127.0.0.1", "--master-port", "29545", os.path.abspath(__file__)] + sys.argv[1:]
        sys.exit(subprocess.run(cmd).returncode)
    import nerface_oracle as O
    import nerf
    from nerf import _engine, fused_train, ray_sampler

    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(0)  # every rank alike: the graphs' device draws
    H = W = 512
    n_img = a.images
    frs = [O.synthetic_frame(i, H, W) for i in range(n_img)]
    g = torch.Generator().manual_seed(1)
    images = torch.rand(n_img, H, W, 3, generator=g).to(dev)
    bg = frs[0]["bg"].to(dev)
    bboxs = [(150 + 4 * i, 400, 128, 380 - 3 * i) for i in range(n_img)]
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs]).to(dev)
    data = ray_sampler.TrainImages(images, poses, exprs, bboxs, frs[0]["intrinsics"], background=bg, device=dev)
    eng = _engine.renderer_for(dev)

    def trainer():
        mk = lambda s: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
            num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
        mc, mf = mk(0), mk(1)
        mc.load_state_dict(O.random_init_params(100))
        mf.load_state_dict(O.random_init_params(101))
        return fused_train.FusedTrainer(mc.to(dev), mf.to(dev), n_latent=n_img, num_coarse=64, num_fine=64, perturb=True, noise_std=0.1)

    rng = torch.Generator().manual_seed(2)
    configs, launches = {}, {}
    # A graph holds the renderer's buffers as sized when it was captured, and a larger call grows (re-allocates) them: size
    # everything with the largest step (weak scaling, then K = 8) and count the eager launches first, then capture.
    # (name, K, rays per image)
    steps = [(f"weak K={world}x2048", world, 2048)] + [(f"K={k}", k, a.rays // k) for k in (8, 4, 2, 1)]
    trainers = {name: trainer() for name, _, _ in steps}
    for name, k, n in steps:
        t = trainers[name]
        t.step_images(data, list(range(k)), n, world=world)
        l0 = eng.launch_count()
        t.step_images(data, list(range(k)), n, world=world)
        launches[name] = eng.launch_count() - l0 + (1 if k == 1 else 0)  # the graph runs Adam's schedule on the device (+1 at K = 1)
    if world == 1:
        smp = ray_sampler.RaySampler(H, W, bboxs, size=a.rays, device=dev)
        tl = trainer().capture(a.rays)

        def loop_step():
            i = int(torch.randint(n_img, (1,), generator=rng))
            s = smp.sample(i, pose=frs[i]["pose"], intrinsics=frs[i]["intrinsics"], image=images[i], background=bg)
            tl.step_graph(s["ray_origins"], s["ray_directions"], s["target"], exprs[i], i, background=s["background"])
        configs["loop"] = loop_step
        l0 = eng.launch_count()
        loop_step()
        launches["loop"] = eng.launch_count() - l0  # outside the graph: the sampler

    for name, k, n in sorted(steps, key=lambda s: (s[0].startswith("weak"), s[1])):
        t = trainers[name]
        t.capture_images(data, k, n, world=world)
        idx = torch.empty(k, dtype=torch.int32).pin_memory()
        configs[name] = (lambda t=t, k=k, idx=idx: (idx.copy_(torch.randint(n_img, (k,), generator=rng, dtype=torch.int32)),
                                                         t.step_images_graph(idx)))

    times = {name: [] for name in configs}
    for _ in range(a.rounds):
        for name, fn in configs.items():
            for _ in range(a.warmup):
                fn()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    if world > 1:
        dist.destroy_process_group()
    if rank != 0:
        return
    res = dict(bench="images_step", card=torch.cuda.get_device_name(dev), power_limit_w=power_limit(), gpus=world, frame=f"{H}x{W}",
               samples="64c+64f", rays_per_step=a.rays, steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               ms_per_step={name: round(statistics.median(v), 3) for name, v in times.items()},
               ms_per_step_all={name: [round(x, 3) for x in v] for name, v in times.items()},
               launches_per_step=launches)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
