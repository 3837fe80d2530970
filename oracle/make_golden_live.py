"""Generate tests/golden/live/*.npz: what the CPU tests that pin this project to the UNMODIFIED reference compare against.

Executes the reference (read-only) on the small inputs those tests define and stores its outputs, so a checkout without the
reference tree still runs every comparison:

  oracle_cases.npz          tests/test_oracle_vs_reference_cpu.py   run_one_iter_of_nerf on six configurations, with its random draws
  backward.npz              tests/test_backward_reference_cpu.py    the training loss's autograd (gradients sampled per tensor)
  dropin_helpers.npz        tests/test_dropin_helpers_cpu.py        ray bundle, encodings, helpers, CfgNode, model class
  dataset.npz               tests/test_dataset_cpu.py               load_flame_data on the synthetic dataset
  products_cuda.npz         tests/test_post_gpu.py                  the eval script's post-render functions on torch CUDA (--cuda;
                                                                   needs a GPU and the reference staged by oracle/stage_reference.py)

Usage:  python oracle/make_golden_live.py [--cuda]
"""
import argparse
import os
import sys
import tempfile
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden", "live")
sys.path.insert(0, HERE)
import golden_io  # noqa: E402
import nerface_oracle as O  # noqa: E402

NEAR, FAR = 0.2, 0.8

# name: (H, W, Sampling(nc, nf, perturb, noise_std, white_bkgd, chunksize), mode, use_bg, use_fine, stress, ablation)
ORACLE_CASES = {
    "min_coarse_3c5f": (3, 4, O.Sampling(3, 5, False, 0.0, False, 65536), "validation", True, True, True, False),
    "one_fine_sample": (2, 5, O.Sampling(64, 1, False, 0.0, False, 65536), "validation", True, True, False, False),
    "ragged_chunks_train": (5, 3, O.Sampling(16, 8, True, 0.2, False, 7), "train", True, True, True, False),
    "perturb_only_white_nobg": (4, 4, O.Sampling(40, 72, True, 0.0, True, 65536), "validation", False, True, True, False),
    "noise_only_coarse_only": (4, 3, O.Sampling(24, 0, False, 0.3, False, 5), "train", True, False, False, False),
    # chunk size divides the ray count: with a ragged last chunk the reference itself raises (every chunk takes the FIRST chunk's
    # ablation directions, train_utils.py:82 — the quirk the oracle and the kernels reproduce)
    "ablation_all_stochastic": (3, 5, O.Sampling(32, 48, True, 0.1, False, 5), "validation", True, True, True, True),
}
# (stress, white, use_bg)
BACKWARD_CASES = {"random_init": (False, False, True), "opaque_stress": (True, False, True), "opaque_stress_white_nobg": (True, True, False)}
GRAD_SAMPLES = 512  # entries of each parameter gradient stored (fixed per tensor name), besides its max |g|


def grad_sample_index(name, numel):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    return np.sort(rng.choice(numel, size=min(numel, GRAD_SAMPLES), replace=False))


def oracle_case_inputs(name):
    H, W, s, mode, use_bg, use_fine, stress, ablation = ORACLE_CASES[name]
    ci = 200 + list(ORACLE_CASES).index(name)
    pc = O.random_init_params(300 + ci, stress)
    pf = O.random_init_params(400 + ci, stress) if use_fine else None
    fr = O.synthetic_frame(ci, H, W)
    fr2 = O.synthetic_frame(ci + 50, H, W) if ablation else None
    return ci, pc, pf, fr, fr2


def backward_inputs(stress, white, use_bg):
    H, W, nc, nf = 2, 5, 64, 64
    s = O.Sampling(nc, nf, True, 0.1, white, 2048)
    fr = O.synthetic_frame(31, H, W)
    pc, pf = O.random_init_params(100, stress), O.random_init_params(101, stress)
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3).clone(), rd.reshape(-1, 3).clone()
    bg = fr["bg"].reshape(-1, 3) if use_bg else None
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(5))
    return H, W, s, fr, pc, pf, ro, rd, bg, target


def dropin_pose(seed):
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
    p = torch.eye(4)
    p[:3, :3] = q
    p[:3, 3] = torch.randn(3, generator=g) * 0.3
    return p


RAY_BUNDLE_CASES = [(7, 5, [1200.0, 1250.0, 0.5, 0.5]), (4, 9, [-900.0, 910.0, 0.48, 0.53]), (16, 16, [333.3, -444.4, 0.1, 0.9])]
PE_CASES = [(10, True, True), (4, False, True), (6, True, False), (1, False, True), (0, True, True)]
MODEL_KW = dict(num_layers=8, hidden_size=256, skip_connect_every=3, num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                include_input_xyz=True, include_input_dir=False, use_viewdirs=True, include_expression=True, latent_code_dim=32)
# a config tree shaped like the scripts' YAML (nested blocks, ints, floats, bools, strings, lists)
CFG_RAW = {
    "experiment": {"id": "synthetic", "logdir": "logs", "randomseed": 42, "train_iters": 1000000, "validate_every": 100,
                   "save_every": 5000, "print_every": 100},
    "dataset": {"type": "blender", "basedir": "data/person", "no_ndc": True, "near": 0.2, "far": 0.8, "testskip": 1,
                "half_res": False, "white_background": False},
    "models": {"coarse": {"type": "ConditionalBlendshapePaperNeRFModel", "num_layers": 8, "hidden_size": 256,
                          "skip_connect_every": 3, "include_input_xyz": True, "num_encoding_fn_xyz": 10},
               "fine": {"type": "ConditionalBlendshapePaperNeRFModel", "num_layers": 8, "hidden_size": 256}},
    "optimizer": {"type": "Adam", "lr": 5.0e-4},
    "scheduler": {"lr_decay": 250, "lr_decay_factor": 0.1},
    "nerf": {"use_viewdirs": True, "encode_position_fn": "positional_encoding",
             "train": {"num_random_rays": 2048, "chunksize": 2048, "perturb": True, "num_coarse": 64, "num_fine": 64,
                       "white_background": False, "radiance_field_noise_std": 0.1, "lindisp": False},
             "validation": {"chunksize": 65536, "perturb": False, "num_coarse": 64, "num_fine": 64, "white_background": False,
                            "radiance_field_noise_std": 0.0, "lindisp": False, "img_size": [512, 512]}},
}
DATASET_CALLS = [dict(half_res=False, testskip=1, test=True), dict(half_res=True, testskip=1), dict(half_res=False, testskip=2)]


def _writer():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_synthetic_dataset", os.path.join(ROOT, "tools", "make_synthetic_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def products_inputs(H, dev):
    gen = torch.Generator().manual_seed(H)
    d = (torch.rand(H, H, generator=gen) * 4 + 1).to(dev)
    w = (torch.rand(H, H, generator=gen) ** 3).to(dev)
    c = torch.rand(H, H, 3, generator=gen).to(dev) * 1.2 - 0.1
    intr = np.array([1200.0 * H / 512, 1150.0 * H / 512, 0.52, 0.47])
    return d, w, c, intr


PRODUCT_SIZES = (64, 512)
PRODUCT_SAMPLES = 16384  # pixels stored of an image with more (a fixed sample); all pixels of a smaller one


def product_sample_index(n_pix):
    if n_pix <= PRODUCT_SAMPLES:
        return np.arange(n_pix)
    return np.sort(np.random.default_rng(n_pix).choice(n_pix, size=PRODUCT_SAMPLES, replace=False))


def product_sample(img):
    """(index, values): a fixed sample of the pixels of an [h, w] or [h, w, c] image, as rows of [h * w, c]."""
    img = np.asarray(img)
    flat = img.reshape(img.shape[0] * img.shape[1], -1)
    idx = product_sample_index(flat.shape[0])
    return idx, flat[idx]


# ------------------------------------------------------------------------------------------------ generators
def gen_oracle_cases(ref, rl):
    import make_golden as MG
    out = {}
    for name, (H, W, s, mode, use_bg, use_fine, stress, ablation) in ORACLE_CASES.items():
        ci, pc, pf, fr, fr2 = oracle_case_inputs(name)
        ro, rd = ref.get_ray_bundle(H, W, np.array(fr["intrinsics"]), fr["pose"][:3, :4])
        ray_bundle = (ro.clone(), rd.clone())
        if mode == "train":
            ro, rd = ro.reshape(-1, 3).clone(), rd.reshape(-1, 3).clone()
        bg = fr["bg"].reshape(-1, 3) if use_bg else None
        rd_abl = ref.get_ray_bundle(H, W, np.array(fr2["intrinsics"]), fr2["pose"][:3, :4])[1] if ablation else None
        mc = rl.build_model(ref, pc)
        mf = rl.build_model(ref, pf) if use_fine else None
        cfg = rl.make_cfg(ref, s.num_coarse, s.num_fine, s.perturb, s.noise_std, s.white_bkgd, s.chunksize, mode, NEAR, FAR)
        torch.manual_seed(4321 + ci)
        with torch.no_grad(), MG.Recorder() as rec:
            want = ref.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro.clone(), rd.clone(), cfg, mode=mode,
                                            encode_position_fn=ref.get_embedding_function(10, True, True),
                                            encode_direction_fn=ref.get_embedding_function(4, False, True),
                                            expressions=fr["expr"], background_prior=bg, latent_code=fr["latent"],
                                            ray_directions_ablation=rd_abl)
        out[name] = {"ray_bundle": ray_bundle, "rd_ablation": rd_abl, "want": list(want), "draws": [t for _, t in rec.draws]}
    return out


def gen_backward(ref, rl):
    import make_golden as MG
    PARAM_ORDER = [k for k in O.random_init_params(100).keys()]
    out = {}
    orig_relu = torch.nn.functional.relu
    torch.nn.functional.relu = lambda x, *a, **k: orig_relu(x).clone()  # the gradient-baseline patch (ref_loader docstring)
    try:
        for tag, (stress, white, use_bg) in BACKWARD_CASES.items():
            H, W, s, fr, pc, pf, ro, rd, bg, target = backward_inputs(stress, white, use_bg)
            ro_r, rd_r = ref.get_ray_bundle(H, W, np.array(fr["intrinsics"]), fr["pose"][:3, :4])
            assert torch.equal(ro_r.reshape(-1, 3), ro) and torch.equal(rd_r.reshape(-1, 3), rd)
            mc, mf = rl.build_model(ref, pc), rl.build_model(ref, pf)
            lat = fr["latent"].clone().requires_grad_(True)
            cfg = rl.make_cfg(ref, s.num_coarse, s.num_fine, True, 0.1, white, 2048, "train", NEAR, FAR)
            torch.manual_seed(77)
            with MG.Recorder() as rec:
                o = ref.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro.clone(), rd.clone(), cfg, mode="train",
                                             encode_position_fn=ref.get_embedding_function(10, True, True),
                                             encode_direction_fn=ref.get_embedding_function(4, False, True),
                                             expressions=fr["expr"], background_prior=bg, latent_code=lat)
            loss = torch.nn.functional.mse_loss(o[0][..., :3], target) + torch.nn.functional.mse_loss(o[3][..., :3], target)
            loss.backward()
            grads = {}
            for net, model in (("coarse", mc), ("fine", mf)):
                named = dict(model.named_parameters())
                for k in PARAM_ORDER:
                    g = named[k].grad
                    if g is None:
                        grads[f"{net}/{k}"] = None
                        continue
                    flat = g.reshape(-1)
                    idx = grad_sample_index(f"{net}/{k}", flat.numel())
                    grads[f"{net}/{k}"] = {"index": idx, "value": flat[torch.from_numpy(idx)].clone(),
                                           "absmax": float(flat.abs().max()), "shape": list(g.shape)}
            out[tag] = {"out": [t.detach() for t in o], "draws": [t for _, t in rec.draws], "loss": float(loss.detach()),
                        "grads": grads, "latent_grad": lat.grad.clone()}
    finally:
        torch.nn.functional.relu = orig_relu
    return out


def gen_dropin(ref):
    out = {"ray_bundle": [], "pe": [], "embedding": []}
    for H, W, intr in RAY_BUNDLE_CASES:
        out["ray_bundle"].append(ref.get_ray_bundle(H, W, np.array(intr), dropin_pose(H * 100 + W)[:3, :4]))
    for n_freq, inc, log in PE_CASES:
        x = torch.randn(37, 3, generator=torch.Generator().manual_seed(n_freq)) * 3.0
        out["pe"].append(ref.positional_encoding(x, n_freq, inc, log))
        out["embedding"].append(ref.get_embedding_function(n_freq, inc, log)(x))
    a, b = torch.arange(5, dtype=torch.float32), torch.arange(3, dtype=torch.float32) * 2.0
    out["meshgrid"] = list(ref.meshgrid_xy(a, b))
    x = torch.randn(23, 4, generator=torch.Generator().manual_seed(3))
    out["minibatches"] = [list(ref.get_minibatches(x, chunksize=cs)) for cs in (1, 7, 23, 100)]
    y = torch.randn(23, 4, generator=torch.Generator().manual_seed(4))
    out["img2mse"] = ref.img2mse(x, y)
    out["mse2psnr"] = [ref.mse2psnr(m) for m in (0.0, 1e-5, 0.0123, 1.0)]
    import yaml
    cfg = ref.CfgNode(CFG_RAW)

    def leaves(node, trail):
        res = []
        for k in node.keys():
            v = getattr(node, k)
            if isinstance(v, dict):
                res.append([trail + [k], "dict", type(v).__name__])
                res += leaves(v, trail + [k])
            else:
                res.append([trail + [k], type(v).__name__, v])
        return res
    out["cfg_leaves"] = leaves(cfg, [])
    out["cfg_dump_roundtrip_equal"] = yaml.safe_load(cfg.dump()) == CFG_RAW
    torch.manual_seed(11)
    m = ref.models.ConditionalBlendshapePaperNeRFModel(**MODEL_KW)
    out["state_dict"] = [[k, list(v.shape), str(v.dtype)] for k, v in m.state_dict().items()]
    out["attributes"] = {n: getattr(m, n) for n in ("dim_xyz", "dim_dir", "dim_expression", "dim_latent_code", "use_viewdirs")}
    out["numel"] = sum(p.numel() for p in m.parameters())
    m.load_state_dict(O.random_init_params(100), strict=True)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(19, m.dim_xyz + m.dim_dir, generator=g)
    expr, lat = torch.randn(76, generator=g), torch.randn(32, generator=g)
    with torch.no_grad():
        out["forward"] = m(x, expr, lat)
    return out


def gen_dataset(ref):
    import cv2
    sys.modules["imageio"].imread = lambda p: cv2.imread(p, cv2.IMREAD_UNCHANGED)[..., ::-1]
    with tempfile.TemporaryDirectory() as d:
        _writer().write_dataset(d, 32, 3, 1, 4)
        return [list(ref.load_flame_data(d, **kw)) for kw in DATASET_CALLS]


def gen_products_cuda(ev):
    dev = torch.device("cuda", 0)
    out = {}
    for H in PRODUCT_SIZES:
        d, w, c, intr = products_inputs(H, dev)
        ref_n = ev.torch_normal_map(d.clone(), intr, w.clone(), clean=True).cpu().numpy().astype("uint8")
        ref_d = np.asarray(ev.cast_to_disparity_image(d))
        ref_c = np.asarray(ev.cast_to_image(c, "blender"))
        out[str(H)] = {name: {"shape": list(img.shape), "sample": list(product_sample(img))}
                       for name, img in (("rgb", ref_c), ("normals", ref_n), ("disparity", ref_d))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", action="store_true", help="only the post-render products on torch CUDA")
    a = ap.parse_args()
    import ref_loader as rl
    assert torch.get_float32_matmul_precision() == "highest"
    if a.cuda:
        ev = rl.load_eval_script()
        assert ev is not None, "no reference tree: run oracle/stage_reference.py first"
        golden_io.save(os.path.join(GOLDEN, "products_cuda.npz"), gen_products_cuda(ev))
        return
    ref = rl.load_reference()
    assert ref is not None, "no reference tree"
    golden_io.save(os.path.join(GOLDEN, "oracle_cases.npz"), gen_oracle_cases(ref, rl))
    golden_io.save(os.path.join(GOLDEN, "dropin_helpers.npz"), gen_dropin(ref))
    golden_io.save(os.path.join(GOLDEN, "dataset.npz"), gen_dataset(ref))
    golden_io.save(os.path.join(GOLDEN, "backward.npz"), gen_backward(ref, rl))


if __name__ == "__main__":
    main()
