"""First-light diagnostic for the fused kernel (run on an H100): compares every stage the kernel can dump
(sample depths, positional encoding, each layer's activations, raw MLP outputs, the seven outputs) with the CPU
oracle.  Usage: python tools/gpu_diag.py [fast|exact] [--stress]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import nerface_oracle as O  # noqa: E402
import nerf  # noqa: E402
from nerf import _engine  # noqa: E402


def main():
    prec = "exact" if "exact" in sys.argv else "fast"
    stress = "--stress" in sys.argv
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    H = W = 8
    fr = O.synthetic_frame(0, H, W)
    pc, pf = O.random_init_params(100, stress), O.random_init_params(101, stress)
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3).contiguous(), rd.reshape(-1, 3).contiguous()
    bg = fr["bg"].reshape(-1, 3)
    s = O.Sampling(64, 128, False, 0.0, False, 65536)
    ex = {}
    rays = torch.cat((ro, rd, torch.full((64, 1), 0.2), torch.full((64, 1), 0.8)), dim=-1)
    with torch.no_grad():
        ref = O.render_chunk(rays, pc, pf, s, fr["expr"], fr["latent"], bg, O.Noise(), extras=ex)
    mc = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                         include_input_xyz=True, include_input_dir=False).to(dev)
    mf = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                         include_input_xyz=True, include_input_dir=False).to(dev)
    mc.load_state_dict(pc)
    mf.load_state_dict(pf)
    eng = _engine.renderer_for(dev)
    eng.sync_weights(mc, mf)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    kw = dict(near=0.2, far=0.8, num_coarse=64, num_fine=128, background=bg.to(dev), precision=prec)
    # oracle per-layer activations for the first 128 coarse rows (rays 0,1)
    pts = ro[:2, None, :] + rd[:2, None, :] * ex["z_coarse"][:2, :, None]
    x = O._encode(pts, rays[:2, 5:8])
    acts = O.mlp_activations(pc, x, fr["expr"], fr["latent"])
    print(f"== precision {prec} stress={stress}")
    for step in [-1] + list(range(9)):
        out = eng.render(ro.to(dev), rd.to(dev), debug=True, act_step=step, **kw)
        torch.cuda.synchronize()
        got = out["act"].cpu()
        if step == -1:
            want = x[:, :63]
            g = got[:, :63]
        else:
            want = acts[step]
            g = got[:, :want.shape[1]]
        err = (g - want).abs()
        print(f"step {step:2d}: max|d| {float(err.max()):.3e}  mean|d| {float(err.mean()):.3e}  ref max {float(want.abs().max()):.3e}"
              f"  worst row {int(err.max(dim=1).values.argmax())} col {int(err.max(dim=0).values.argmax())}")
    out = eng.render(ro.to(dev), rd.to(dev), debug=True, **kw)
    torch.cuda.synchronize()
    for k, want in (("z_coarse", ex["z_coarse"]), ("raw_coarse", None), ("z_fine", ex["z_fine"]), ("raw_fine", None)):
        got = out[k].cpu()
        if want is None:
            # raw dumps are taken before the background overwrite: compare sigma and the non-last rgb
            want = ex[k]
            d = (got - want).abs()
            d[:, -1, :3] = 0
            print(f"{k:10s}: max|d| {float(d.max()):.3e}  (sigma {float(d[..., 3].max()):.3e})  ref max {float(want.abs().max()):.3e}")
        else:
            print(f"{k:10s}: max|d| {float((got - want).abs().max()):.3e}")
    names = ["rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last"]
    for nme, want in zip(names, ref):
        print(f"{nme:11s}: max|d| {float((out[nme].cpu() - want).abs().max()):.3e}   ref range [{float(want.min()):.3f},{float(want.max()):.3f}]")
    print("launches", eng.launch_count())


if __name__ == "__main__":
    main()
