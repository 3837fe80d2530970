#!/usr/bin/env python
"""SHA-256 digests of everything the library computes on fixed, seeded inputs, for comparing two builds bit for bit (a
refactor of the kernels or of the host layer must leave every digest and the launch count unchanged):

  eval     64c+128f evaluation render of 2304 rays with a background: the seven outputs
  train    2048 rays at 64c+64f, stratified sampling, sigma noise 0.1, background, dir_z: the seven outputs of the training
           forward, all 48 parameter gradients, the latent gradient and the five input gradients
  chunked  the same for 200 rays with NFB_TRAIN_MEM_MB=48 (32 rays per chunk, the last chunk ragged)

each in both precision modes, plus the launches each case took.  Usage:

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

    def train_case(case, n, prec, seed):
        g = torch.Generator().manual_seed(seed)
        nz = O.draw_noise(n, O.Sampling(64, 64, True, 0.1, False, 2048), g)
        noise = {k: getattr(nz, k).to(dev) for k in ("t_rand", "n_c", "u", "n_f")}
        dz = (torch.rand(n, generator=g) * 2.0 - 1.0).to(dev)
        shapes = [(n, 3), (n,), (n,), (n, 3), (n,), (n,), (n,)]
        gouts = [((torch.rand(sh, generator=g) - 0.3) / n).to(dev) for sh in shapes]
        l0 = eng.launch_count()
        out = eng.render(ro[:n].contiguous(), rd[:n].contiguous(), NEAR, FAR, 64, 64, perturb=True, noise_std=0.1,
                         background=bg[:n].contiguous(), dir_z=dz, noise=noise, precision=prec, train=True)
        gc, gf, gl, ing = eng.backward(gouts, pc, pf, want_latent=True, want_params=True, inputs=INPUTS)
        named = [(k, out[k]) for k in OUTPUTS]
        named += [(f"grad_coarse/{PARAM_ORDER[i]}", t) for i, t in enumerate(gc) if t is not None]
        named += [(f"grad_fine/{PARAM_ORDER[i]}", t) for i, t in enumerate(gf) if t is not None]
        named += [("grad_latent", gl)] + [("grad_" + k, t) for k, t in sorted(ing.items())]
        record(case, named, l0)

    for prec in ("fast", "exact"):
        l0 = eng.launch_count()
        out = eng.render(ro, rd, NEAR, FAR, 64, 128, background=bg, precision=prec)
        record(f"eval/{prec}", [(k, out[k]) for k in OUTPUTS], l0)
        train_case(f"train/{prec}", 2048, prec, 1031)
        os.environ["NFB_TRAIN_MEM_MB"] = "48"  # read by the library on every call
        try:
            train_case(f"chunked/{prec}", 200, prec, 1032)
        finally:
            del os.environ["NFB_TRAIN_MEM_MB"]

    res["device"] = torch.cuda.get_device_name(0)
    with open(sys.argv[1], "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"{sum(len(v) - 1 for v in res.values() if isinstance(v, dict))} digests -> {sys.argv[1]}")


if __name__ == "__main__":
    main()
