"""Worker of tests/test_multigpu_images.py — run under torch.distributed.run with one rank per GPU (NCCL).  Data-parallel steps
over several images and data_parallel(nerf.render_frames), each compared across the ranks and with the same work done by ONE
GPU in the same process; rank 0 prints `MGPU_OK <name>` per check."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "4d-facial-avatars_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import nerface_oracle as O  # noqa: E402
import nerf  # noqa: E402
from nerf import fused_train, parallel, ray_sampler  # noqa: E402

N_IMAGES = 6
# C3's gate of test_sharded_fp64_gpu.py (test_backward_fp64_gpu.TOL, fast mode) holds each side against float64, so two sides
# differ by at most twice it: (max error / max |ref|, relative L2) per tensor.
GATE = (2 * 4e-2, 2 * 3e-2)


def make_model(params, dev):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    m.load_state_dict(params)
    return m.to(dev)


def within_gate(a, b, tag):
    a, b = a.double(), b.double()
    m = float(b.abs().max())
    if m == 0.0:
        assert float(a.abs().max()) == 0.0, tag
        return
    em, el = float((a - b).abs().max()) / m, float((a - b).norm() / b.norm())
    assert em <= GATE[0] and el <= GATE[1], (tag, em, el)


def same_on_every_rank(t, tag):
    ref = t.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(ref, t), tag


def main():
    world, rank, local = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    ok = lambda name: rank == 0 and print("MGPU_OK", name, flush=True)  # noqa: E731

    H = W = 64
    frs = [O.synthetic_frame(40 + i, H, W) for i in range(N_IMAGES)]
    g = torch.Generator().manual_seed(140)
    images = torch.rand(N_IMAGES, H, W, 3, generator=g).to(dev)
    data = ray_sampler.TrainImages(images, torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs]),
                                   torch.stack([f["expr"] for f in frs]), [(4 + 2 * i, 60, 2 + i, 62 - i) for i in range(N_IMAGES)],
                                   frs[0]["intrinsics"], background=frs[0]["bg"], device=dev)
    lat0 = torch.randn(N_IMAGES, 32, generator=torch.Generator().manual_seed(3)) * 0.1

    def trainer():
        return fused_train.FusedTrainer(make_model(O.random_init_params(100), dev), make_model(O.random_init_params(101), dev),
                                        n_latent=N_IMAGES, num_coarse=64, num_fine=64, perturb=True, noise_std=0.1, latent_codes=lat0)

    # ---- 1. K-image steps over the ranks: the summed bucket against one GPU, then 5 eager and 5 captured steps in lock-step
    k, n, rounds = 4, 256, 32
    gen = torch.Generator(device=dev).manual_seed(7)  # the same draws on every rank
    draws = torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=gen)
    ids = [0, 3, 3, 5]
    tr, one = trainer(), trainer()
    for t, w, r in ((tr, world, rank), (one, 1, 0)):
        t._own_engine()
        sb = t._images_buffers(data, k, n)
        sb["img"].copy_(torch.tensor(ids, dtype=torch.int32))
        t._images_sample(data, sb, n, draws, rounds)
        torch.manual_seed(11)
        t._images_gradients(sb, k, n, w, r)
        if w > 1:
            dist.all_reduce(t.grads)
            t._images_regulariser(sb, k)
    torch.cuda.synchronize()
    same_on_every_rank(tr.grads, "bucket")
    for i, (a, b) in enumerate(zip(tr._gviews, one._gviews)):
        within_gate(a, b, ("param", i))
    within_gate(tr.grads[tr.lat_off:], one.grads[one.lat_off:], "latent rows")
    tr.grads.zero_()
    for i in range(5):
        torch.manual_seed(100 + i)
        tr.step_images(data, [(i + j) % N_IMAGES for j in range(k)], n, draws=torch.rand(k * rounds * n, dtype=torch.float64,
                       device=dev, generator=gen), max_rounds=rounds, world=world)
    tr.capture_images(data, k, n, max_rounds=rounds, device_draws=False, world=world)
    for i in range(5):
        tr.step_images_graph([(2 * i + j) % N_IMAGES for j in range(k)],
                             draws=torch.rand(k * rounds * n, dtype=torch.float64, device=dev, generator=gen))
    torch.cuda.synchronize()
    for name in ("params", "exp_avg", "exp_avg_sq"):
        same_on_every_rank(getattr(tr, name), name)
    assert tr.iter == 10 and bool(torch.isfinite(tr.params).all())
    ok("images_steps_lockstep")

    # ---- 2. data_parallel(nerf.render_frames): outputs bit for bit the unsharded call's, gradients within the gate
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=65536)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk, validation=blk), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    fr = frs[0]
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(dev))
    sel = torch.randperm(H * W, generator=torch.Generator().manual_seed(5))[:512].to(dev)
    ro, rd = ro.reshape(-1, 3)[sel], rd.reshape(-1, 3)[sel]
    bg = fr["bg"].reshape(-1, 3).to(dev)[sel]
    fi = torch.randint(0, 3, (512,), generator=torch.Generator().manual_seed(6), dtype=torch.int32).to(dev)
    expr = data.expressions[:3]
    tgt = images[0].reshape(-1, 3)[sel]
    fids = torch.tensor([1, 4, 4], device=dev)
    dp = parallel.data_parallel(nerf.render_frames)
    with torch.no_grad():
        for mode in ("validation", "train"):
            mc, mf = make_model(O.random_init_params(100), dev), make_model(O.random_init_params(101), dev)
            torch.manual_seed(21)
            a = nerf.render_frames(ro, rd, fi, expr, lat0[:3].to(dev), mc, mf, cfg, mode=mode, background_prior=bg)
            torch.manual_seed(21)
            b = dp(ro, rd, fi, expr, lat0[:3].to(dev), mc, mf, cfg, mode=mode, background_prior=bg)
            assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b)), mode

    def grads_of(run, shard):
        mc, mf = make_model(O.random_init_params(100), dev), make_model(O.random_init_params(101), dev)
        table = lat0.clone().to(dev).requires_grad_(True)
        torch.manual_seed(22)
        out = run(ro, rd, fi, expr, table[fids], mc, mf, cfg, mode="train", background_prior=bg)
        loss = ((out[0] - tgt) ** 2).mean() + ((out[3] - tgt) ** 2).mean() + 0.005 / 3 * sum(table[i].norm() for i in fids)
        loss.backward()
        params = list(mc.parameters()) + list(mf.parameters()) + [table]
        if shard:
            parallel.allreduce_gradients(params, average=True)
        return [p.grad.clone() for p in params if p.grad is not None], [o.detach() for o in out]
    g1, o1 = grads_of(nerf.render_frames, False)
    g2, o2 = grads_of(dp, True)
    assert all(torch.equal(x, y) for x, y in zip(o1, o2) if x is not None)
    for i, (a, b) in enumerate(zip(g2, g1)):
        within_gate(a, b, ("render_frames grad", i))
    ok("dp_render_frames")

    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
