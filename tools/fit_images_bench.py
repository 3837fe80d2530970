#!/usr/bin/env python
"""Fitting-step benchmark over several images (DESIGN.md 8d): a frozen avatar's per-image pose, expression and latent fitted
to 512x512 synthetic frames, 64 coarse + 64 fine samples, stratified sampling + sigma noise 0.1, 2048 rays per step in all
(2048 / K per image), at K = 1, 2 and 8 images per step.  Three ways of taking one step, alternated in one process:

  (a) dropin — tools/fit_bench.py's loop over K frames: get_ray_bundle over every frame's whole H x W from a requires_grad pose,
               indexed down to the sampled pixels, nerf.render_frames, torch MSE, loss.backward() through autograd and
               torch.optim.Adam with one parameter group per table (the pixels are FusedFitter's, drawn beforehand);
  (b) eager  — FusedFitter.step;
  (c) graph  — FusedFitter.step_graph (one CUDA graph replay per step).

Learning rates are FusedFitter's defaults (1e-4 per table).  Per configuration: --warmup steps, then --steps steps between two
CUDA events, --rounds times in turn; the median ms per step is reported, with the card's name and power limit read in the same
process and the library's launches per step (nfb_launch_count over one eager step).  --profile runs instead, in a run of its
own, torch.profiler over --steps steps of each configuration and prints the GPU time per step of every kernel."""
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        w, mhz = out.splitlines()[0].split(",")
        return float(w), float(mhz)
    except Exception:  # noqa: BLE001  (no nvidia-smi: the numbers are reported without it)
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--rays", type=int, default=2048)
    ap.add_argument("--ks", default="1,2,8")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import nerface_oracle as O
    import nerf
    from nerf import _engine

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    H = W = 512
    n_img = a.images
    frs = [O.synthetic_frame(i, H, W) for i in range(n_img)]
    g = torch.Generator().manual_seed(1)
    images = torch.rand(n_img, H, W, 3, generator=g).to(dev)
    bg = frs[0]["bg"].to(dev)
    bboxs = [(150 + 4 * i, 400, 128, 380 - 3 * i) for i in range(n_img)]
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs])
    lats = torch.stack([f["latent"] for f in frs])
    intr = frs[0]["intrinsics"]
    mk = lambda s: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(0), mk(1)
    mc.load_state_dict(O.random_init_params(100))
    mf.load_state_dict(O.random_init_params(101))
    mc, mf = mc.to(dev).requires_grad_(False), mf.to(dev).requires_grad_(False)
    eng = _engine.renderer_for(dev)
    rng = torch.Generator().manual_seed(2)
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=1 << 20)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))

    def fitter():
        return nerf.FusedFitter(mc, mf, images, bboxs, intr, poses, exprs, lats, background=bg)

    def pick(k):
        return [int(i) for i in torch.randint(n_img, (k,), generator=rng)]

    configs, launches, fitters = {}, {}, {}
    ks = [int(v) for v in a.ks.split(",")]
    for k in sorted(ks, reverse=True):  # the largest step first: later graphs never see their buffers re-allocated
        n = a.rays // k
        f = fitters[k] = fitter()
        f.step(list(range(k)), n)
        l0 = eng.launch_count()
        f.step(list(range(k)), n)
        launches[f"K={k}"] = eng.launch_count() - l0

        # (a) the drop-in loop over K frames: its own leaves and torch.optim.Adam (three groups), pixels drawn by the fitter's sampler
        P = poses.clone().to(dev).requires_grad_(True)
        E = exprs.clone().to(dev).requires_grad_(True)
        L = lats.clone().to(dev).requires_grad_(True)
        opt = torch.optim.Adam([dict(params=[P], lr=f.lr["pose"]), dict(params=[E], lr=f.lr["expression"]),
                                dict(params=[L], lr=f.lr["latent"])])
        sel = f._bufs[(k, n, True)]

        def dropin(k=k, n=n, P=P, E=E, L=L, opt=opt, sel=sel):
            ids = torch.tensor(pick(k), device=dev)
            rc = sel["pixel_rc"].long()
            flat = (rc[:, 0] * W + rc[:, 1]).view(k, n)
            ro, rd = [], []
            for j in range(k):
                o, d = nerf.get_ray_bundle(H, W, intr, P[ids[j]].view(3, 4))
                ro.append(o.reshape(-1, 3)[flat[j]])
                rd.append(d.reshape(-1, 3)[flat[j]])
            out = nerf.render_frames(torch.cat(ro), torch.cat(rd), sel["frame_index"], E[ids], L[ids], mc, mf, cfg, mode="train",
                                     background_prior=sel["background"])
            loss = (torch.nn.functional.mse_loss(out[0], sel["target"]) + torch.nn.functional.mse_loss(out[3], sel["target"])
                    + (f.latent_reg / k) * sum(torch.norm(L[i]) for i in ids))
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()

        configs[f"dropin K={k}"] = dropin
        configs[f"eager K={k}"] = (lambda f=f, k=k, n=n: f.step(pick(k), n))
    for k in sorted(ks, reverse=True):
        f = fitters[k]
        f.capture(k, a.rays // k)
        idx = torch.empty(k, dtype=torch.int32).pin_memory()
        configs[f"graph K={k}"] = (lambda f=f, k=k, idx=idx: (idx.copy_(torch.tensor(pick(k), dtype=torch.int32)), f.step_graph(idx)))
    order = [f"{m} K={k}" for k in ks for m in ("dropin", "eager", "graph")]
    watts, mhz = power_limit()
    res = dict(bench="fit_images_step", card=torch.cuda.get_device_name(dev), power_limit_w=watts, max_sm_clock_mhz=mhz, frame=f"{H}x{W}",
               samples="64c+64f", rays_per_step=a.rays, fit="pose+expression+latent", steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               launches_per_step=launches)

    if a.profile:
        per = {}
        for name in order:
            fn = configs[name]
            for _ in range(a.warmup):
                fn()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.steps):
                    fn()
                torch.cuda.synchronize()
            tot = {}
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    key = e.name.split("(")[0][:80]
                    tot[key] = tot.get(key, 0.0) + getattr(e, "device_time", getattr(e, "cuda_time", 0.0)) / a.steps
            per[name] = {kk: round(v, 1) for kk, v in sorted(tot.items(), key=lambda kv: -kv[1]) if v >= 1.0}
            per[name]["total_us"] = round(sum(tot.values()), 1)
        res["kernels_us_per_step"] = per
        print(json.dumps(res))
        return

    times = {name: [] for name in order}
    for _ in range(a.rounds):
        for name in order:
            fn = configs[name]
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
    res["ms_per_step"] = {name: round(statistics.median(v), 3) for name, v in times.items()}
    res["ms_per_step_all"] = {name: [round(x, 3) for x in v] for name, v in times.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
