"""Generate tests/golden/*.npz by executing the UNMODIFIED reference (read-only, /root/reference).

Runs only where a reference checkout is readable.  For every case it
  1. imports the reference ``nerf`` package with empty stand-ins for the absent, hot-path-unused
     modules (pytorch3d, torchsearchsorted, imageio) — SURVEY.md §8(c);
  2. runs ``run_one_iter_of_nerf`` on seeded synthetic inputs, recording every torch.rand/randn draw
     and every MLP output;
  3. runs oracle/nerface_oracle.py on the same inputs + recorded noise and prints the max-abs gap;
  4. writes inputs, noise and the REFERENCE's outputs to tests/golden/<case>.npz.

Usage:  python oracle/make_golden.py [--ref /root/reference]
"""
import argparse
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import nerface_oracle as O  # noqa: E402


def import_reference(ref_root):
    for name in ("pytorch3d", "pytorch3d.transforms", "torchsearchsorted", "imageio"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, os.path.join(ref_root, "nerface_code", "nerf-pytorch"))
    import nerf  # the reference package
    return nerf


class Recorder:
    """Records torch.rand / torch.randn draws made inside the reference."""

    def __init__(self):
        self.draws = []
        self._rand, self._randn = torch.rand, torch.randn

    def __enter__(self):
        def rand(*a, **k):
            t = self._rand(*a, **k)
            self.draws.append(("rand", t.clone()))
            return t

        def randn(*a, **k):
            t = self._randn(*a, **k)
            self.draws.append(("randn", t.clone()))
            return t

        torch.rand, torch.randn = rand, randn
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randn = self._rand, self._randn


def make_cfg(nerf, s: O.Sampling, mode, near, far):
    blk = dict(num_coarse=s.num_coarse, num_fine=s.num_fine, perturb=s.perturb, lindisp=False,
               radiance_field_noise_std=s.noise_std, white_background=s.white_bkgd, chunksize=s.chunksize)
    return nerf.CfgNode(dict(nerf={"use_viewdirs": True, mode: blk}, dataset=dict(no_ndc=True, near=near, far=far)))


def build_model(nerf, params):
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False,
        use_viewdirs=True, include_expression=True, latent_code_dim=32)
    m.load_state_dict(params)
    return m


CASES = {
    # name: (H, W, Sampling, mode, use_bg, use_fine, stress, ablation)
    "det_64c128f": (8, 8, O.Sampling(64, 128, False, 0.0, False, 65536), "validation", True, True, False, False),
    "det_stress_64c128f": (8, 8, O.Sampling(64, 128, False, 0.0, False, 65536), "validation", True, True, True, False),
    "stoch_train_64c64f": (6, 8, O.Sampling(64, 64, True, 0.1, False, 2048), "train", True, True, False, False),
    "stoch_stress_chunks": (6, 8, O.Sampling(64, 128, True, 0.1, False, 16), "validation", True, True, True, False),
    "coarse_only_32": (8, 8, O.Sampling(32, 0, False, 0.0, False, 65536), "validation", False, False, False, False),
    "det_128c256f": (4, 4, O.Sampling(128, 256, False, 0.0, False, 65536), "validation", True, True, True, False),
    "ablation_dirs": (8, 8, O.Sampling(64, 128, False, 0.0, False, 32), "validation", True, True, True, True),
    "white_nobg": (4, 8, O.Sampling(64, 64, False, 0.0, True, 65536), "validation", False, True, True, False),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(HERE, "..", "tests", "golden"))
    args = ap.parse_args()
    assert torch.get_float32_matmul_precision() == "highest"
    nerf = import_reference(args.ref)
    os.makedirs(args.out, exist_ok=True)
    near, far = 0.2, 0.8
    worst = 0.0
    for ci, (name, (H, W, s, mode, use_bg, use_fine, stress, ablation)) in enumerate(CASES.items()):
        pc = O.random_init_params(100, stress)
        pf = O.random_init_params(101, stress) if use_fine else None
        fr = O.synthetic_frame(ci, H, W)
        ro, rd = nerf.get_ray_bundle(H, W, np.array(fr["intrinsics"]), fr["pose"][:3, :4])
        o_ro, o_rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
        ray_gap = max(float((ro - o_ro).abs().max()), float((rd - o_rd).abs().max()))
        if mode == "train":  # the trainer passes flat gathered rays (train_transformed_rays.py:320-326)
            ro, rd = ro.reshape(-1, 3).clone(), rd.reshape(-1, 3).clone()
        bg = fr["bg"].reshape(-1, 3) if use_bg else None
        rd_abl = None
        if ablation:
            fr2 = O.synthetic_frame(ci + 50, H, W)
            _, rd_abl = nerf.get_ray_bundle(H, W, np.array(fr2["intrinsics"]), fr2["pose"][:3, :4])
        mc = build_model(nerf, pc)
        mf = build_model(nerf, pf) if use_fine else None
        raws = []
        for m in (mc, mf):
            if m is not None:
                m.register_forward_hook(lambda _m, _i, out: raws.append(out.detach().clone()))
        cfg = make_cfg(nerf, s, mode, near, far)
        enc_xyz = nerf.get_embedding_function(10, True, True)
        enc_dir = nerf.get_embedding_function(4, False, True)
        torch.manual_seed(1234 + ci)
        with torch.no_grad(), Recorder() as rec:
            ref = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro.clone(), rd.clone(), cfg, mode=mode,
                                            encode_position_fn=enc_xyz, encode_direction_fn=enc_dir,
                                            expressions=fr["expr"], background_prior=bg, latent_code=fr["latent"],
                                            ray_directions_ablation=rd_abl)
        # split recorded draws back into per-chunk Noise objects (same order the oracle expects)
        n_rays = H * W
        chunks = [min(s.chunksize, n_rays - st) for st in range(0, n_rays, s.chunksize)]
        it = iter(rec.draws)
        noises = []
        for n in chunks:
            nz = O.Noise()
            if s.perturb:
                nz.t_rand = next(it)[1]
            if s.noise_std > 0:
                nz.n_c = next(it)[1]
            if s.num_fine > 0:
                if s.perturb:
                    nz.u = next(it)[1]
                if s.noise_std > 0:
                    nz.n_f = next(it)[1]
            noises.append(nz)
        assert next(it, None) is None, "unconsumed draws"
        with torch.no_grad():
            mine = O.run_one_iter(ro, rd, pc, pf, s, near, far, fr["expr"], fr["latent"], bg, mode,
                                  noise_per_chunk=noises, rd_ablation=rd_abl)
        assert len(ref) == len(mine), (name, len(ref), len(mine))
        gaps = []
        for a, b in zip(ref, mine):
            assert (a is None) == (b is None)
            if a is not None:
                assert a.shape == b.shape, (name, a.shape, b.shape)
                gaps.append(float((a - b).abs().max()))
        worst = max(worst, max(gaps), ray_gap)
        print(f"{name:22s} arity={len(ref)} oracle-vs-reference max|d| per output: "
              + " ".join(f"{g:.2e}" for g in gaps) + f"  rays {ray_gap:.1e}")
        save = dict(H=H, W=W, num_coarse=s.num_coarse, num_fine=s.num_fine, perturb=int(s.perturb),
                    noise_std=s.noise_std, white_bkgd=int(s.white_bkgd), chunksize=s.chunksize,
                    mode=mode, stress=int(stress), near=near, far=far, seed_coarse=100, seed_fine=101,
                    use_fine=int(use_fine), arity=len(ref),
                    param_probe=np.array([float(pc["layers_xyz.3.weight"][7, 300]), float(pc["fc_rgb.bias"][2])]),
                    ro=ro.numpy(), rd=rd.numpy(), expr=fr["expr"].numpy(), latent=fr["latent"].numpy(),
                    pose=fr["pose"].numpy(), intrinsics=np.array(fr["intrinsics"]))
        if bg is not None:
            save["bg"] = bg.numpy()
        if rd_abl is not None:
            save["rd_ablation"] = rd_abl.numpy()
        for k in ("t_rand", "n_c", "u", "n_f"):
            vals = [getattr(nz, k) for nz in noises]
            if vals[0] is not None:
                save["noise_" + k] = torch.cat(vals, dim=0).numpy()
        for i, t in enumerate(ref):
            if t is not None:
                save[f"out{i}"] = t.numpy()
        # MLP outputs in call order: per chunk (coarse, fine) — keep the first chunk's
        save["raw_coarse_chunk0"] = raws[0].numpy()
        if use_fine:
            save["raw_fine_chunk0"] = raws[1].numpy()
        np.savez_compressed(os.path.join(args.out, name + ".npz"), **save)
    print(f"worst oracle-vs-reference gap over all cases: {worst:.3e}")


if __name__ == "__main__":
    main()
