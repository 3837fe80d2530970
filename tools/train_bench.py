#!/usr/bin/env python
"""Training-step benchmark (BASELINE config 3): 2048-ray batches of one synthetic 512x512 frame, 64 coarse + 64 fine
samples (the shipped YAML's train block), stratified sampling + sigma noise, per-frame latent + expression conditioning,
loss = mse(rgb_c) + mse(rgb_f) + 0.005*|latent|, Adam lr 5e-4 — through the drop-in API (run_one_iter_of_nerf in train mode
+ loss.backward() + optimizer.step()).  One process per GPU; with WORLD_SIZE > 1 the ray batch is sharded across ranks
and the gradients are all-reduced in one flat bucket (nerf/parallel.py).

Prints one JSON line: rays/s over the whole step, the split forward / backward / optimizer (CUDA events), and the
tensor-core roofline of the step (3 x 1,100,032 FLOP per MLP evaluation: forward + dX + dW)."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--num-coarse", type=int, default=64)
    ap.add_argument("--num-fine", type=int, default=64)
    ap.add_argument("--precision", default="fast")
    ap.add_argument("--impl", default="fused", choices=["fused", "dropin"],
                    help="fused: nerf/fused_train.py (libnfb launches only); dropin: run_one_iter_of_nerf + torch loss / Adam, as the unmodified script does")
    a = ap.parse_args()
    import nerface_oracle as O
    import nerf
    from nerf import parallel

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    nerf.set_precision(a.precision)
    H = W = 512
    fr = O.synthetic_frame(0, H, W)
    mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(), mk()
    mc.load_state_dict(O.random_init_params(100))
    mf.load_state_dict(O.random_init_params(101))
    mc, mf = mc.to(dev), mf.to(dev)
    latent_codes = torch.zeros(16, 32, device=dev, requires_grad=True)
    params = [p for k, p in list(mc.named_parameters()) + list(mf.named_parameters()) if not k.startswith("layers_dir.3")]
    opt = torch.optim.Adam(params + [latent_codes], lr=5e-4)
    blk = dict(num_coarse=a.num_coarse, num_fine=a.num_fine, perturb=True, lindisp=False, radiance_field_noise_std=0.1,
               white_background=False, chunksize=2048)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(dev))
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    bg = fr["bg"].reshape(-1, 3).to(dev)
    target_img = torch.rand(H * W, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    expr = fr["expr"].to(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    per_rank = a.rays // world
    n_steps = a.steps + a.warmup
    idx = [torch.randint(0, H * W, (a.rays,), device=dev, generator=g) for _ in range(n_steps)]
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(n_steps)]
    eng = nerf._engine.renderer_for(dev)
    trainer = None
    if a.impl == "fused":
        from nerf import fused_train
        trainer = fused_train.FusedTrainer(mc, mf, n_latent=16, lr=5e-4, num_coarse=a.num_coarse, num_fine=a.num_fine, perturb=True,
                                           noise_std=0.1, near=0.2, far=0.8, latent_reg=0.005, precision=a.precision)

    def step_fused(i):
        sel = idx[i][rank * per_rank:(rank + 1) * per_rank]
        ev[i][0].record()
        loss = trainer.gradients(ro[sel], rd[sel], target_img[sel], expr, 3, background=bg[sel], world=world, n_total=a.rays,
                                 events=(ev[i][1], ev[i][2]))
        trainer.update()
        ev[i][3].record()
        return loss.sum()

    def step(i):
        if trainer is not None:
            return step_fused(i)
        sel = idx[i][rank * per_rank:(rank + 1) * per_rank]
        ev[i][0].record()
        out = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro[sel], rd[sel], cfg, mode="train", expressions=expr,
                                        background_prior=bg[sel], latent_code=latent_codes[3])
        tgt = target_img[sel]
        loss = ((out[0] - tgt) ** 2).mean() + ((out[3] - tgt) ** 2).mean() + 0.005 * latent_codes[3].norm()
        ev[i][1].record()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        if world > 1:
            parallel.allreduce_gradients(params + [latent_codes], average=True)
        ev[i][2].record()
        opt.step()
        ev[i][3].record()
        return loss

    losses = []
    for i in range(a.warmup):
        losses.append(float(step(i)))
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    for i in range(a.warmup, n_steps):
        last = step(i)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    losses.append(float(last))
    ms = torch.tensor([sum(ev[i][0].elapsed_time(ev[i][3]) for i in range(a.warmup, n_steps))], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        fwd = sum(ev[i][0].elapsed_time(ev[i][1]) for i in range(a.warmup, n_steps)) / a.steps
        bwd = sum(ev[i][1].elapsed_time(ev[i][2]) for i in range(a.warmup, n_steps)) / a.steps
        ost = sum(ev[i][2].elapsed_time(ev[i][3]) for i in range(a.warmup, n_steps)) / a.steps
        step_ms = float(ms[0]) / a.steps
        evals = 2 * a.num_coarse + a.num_fine
        flop = 3 * 1100032 * evals * a.rays
        peak = 989.0  # H100 SXM data sheet, dense FP16
        pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
        if os.path.exists(pk):
            peak = json.load(open(pk))["bf16_tflops"]
        print(json.dumps({
            "metric": "training rays/sec (2048-ray batches, fwd + bwd + Adam)", "value": a.rays / (step_ms * 1e-3), "unit": "rays/s",
            "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": step_ms,
            "ms_forward_and_loss": fwd, "ms_backward": bwd, "ms_optimizer": ost, "wall_ms_per_step": 1e3 * wall / a.steps,
            "impl": a.impl, "config": {"workload": f"{a.rays} rays/iter, {a.num_coarse}c+{a.num_fine}f, perturb + noise 0.1, Adam", "precision": a.precision,
                       "parallelism": f"dp{world} (ray batch sharded, one flat gradient all-reduce)"},
            "gpu_launches_per_step": (eng.launch_count() - l0) / a.steps,
            "roofline": {"bound": "tensor", "achieved": flop / (step_ms * 1e-3) / 1e12, "peak": peak, "unit": "TFLOP/s",
                         "frac": flop / (step_ms * 1e-3) / 1e12 / peak, "flop_per_step": flop},
            "loss_first_last": [losses[0], losses[-1]]}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
