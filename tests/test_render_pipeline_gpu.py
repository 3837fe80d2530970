"""The render kernel's edge cases of its persistent schedule, bit for bit against a stored run.

The kernel walks a stream of coarse and fine tiles per CTA and hands each unit's per-ray stages (compositing, the CDF,
inverse-CDF sampling, the merge sort, the ray setup) between warps.  These cases put every boundary of that stream under
test: units with an invalid ray (1, 2 and 3 rays), CTAs that run different numbers of units (n_units = k * SMs - 1, k * SMs,
k * SMs + 1), a coarse-only pass (64c+0f, 3c+0f), two coarse tiles per unit (256c+256f), tiles that end inside a ray (3c+7f),
a single one-ray unit (128c+256f), stratified sampling with sigma noise and a background, a white background, and the
chunked training forward.  Each case runs in both precision modes with the per-sample dumps on, and every returned array
is compared by SHA-256 of its bytes with tests/golden/render_pipeline_digests.json.

`python tests/test_render_pipeline_gpu.py` prints the digests of the library it loads (NFB_LIB selects one) in the format
of that file.
"""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "4d-facial-avatars_b200"), os.path.dirname(os.path.abspath(__file__))):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import nerface_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DIGESTS = os.path.join(ROOT, "tests", "golden", "render_pipeline_digests.json")
SMS = 132  # H100 SXM; the digests do not depend on it, only which schedule boundaries the ray counts hit

# name -> (n_rays, nc, nf, options)
CASES = {
    "rays1_64c128f": (1, 64, 128, {}),
    "rays2_64c128f": (2, 64, 128, {}),
    "rays3_64c128f": (3, 64, 128, {}),
    "units_2sm_minus1": (2 * (2 * SMS - 1), 64, 128, {}),
    "units_2sm": (2 * (2 * SMS), 64, 128, {}),
    "units_2sm_plus1": (2 * (2 * SMS + 1), 64, 128, {}),
    "units_2sm_plus1_odd_rays": (2 * (2 * SMS + 1) - 1, 64, 128, {}),
    "coarse_only_64c0f": (2 * SMS + 3, 64, 0, {}),
    "coarse_only_3c0f": (2 * SMS + 3, 3, 0, {}),
    "two_coarse_tiles_256c256f": (SMS + 5, 256, 256, {}),
    "ragged_3c7f": (2 * SMS + 3, 3, 7, {}),
    "one_ray_128c256f": (1, 128, 256, {}),
    "perturb_noise_bg_64c128f": (3 * SMS + 1, 64, 128, {"perturb": True, "noise": True, "bg": True}),
    "white_bkgd_64c128f": (2 * SMS + 1, 64, 128, {"white": True}),
}


def _engine(dev):
    import nerf
    from nerf import _engine
    mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(), mk()
    mc.load_state_dict(O.random_init_params(31, True))
    mf.load_state_dict(O.random_init_params(32, True))
    eng = _engine.renderer_for(dev)
    eng.sync_weights(mc.to(dev), mf.to(dev))
    return eng


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def _rays(n, seed):
    fr = O.synthetic_frame(seed, 32, 32)
    ro, rd = O.ray_bundle(32, 32, fr["intrinsics"], fr["pose"])
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    idx = torch.arange(n) % ro.shape[0]
    return fr, ro[idx].contiguous(), rd[idx].contiguous()


def case_digests(dev, eng, name, prec):
    n, nc, nf, opt = CASES[name]
    fr, ro, rd = _rays(n, 7)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    g = torch.Generator().manual_seed(n * 1000 + nc + nf)
    kw = dict(precision=prec, debug=True)
    if opt.get("perturb"):
        kw["perturb"] = True
        kw["noise_std"] = 1.0
        kw["noise"] = {"t_rand": torch.rand(n, nc, generator=g).to(dev), "n_c": torch.randn(n, nc, generator=g).to(dev),
                       "u": torch.rand(n, nf, generator=g).to(dev), "n_f": torch.randn(n, nc + nf, generator=g).to(dev)}
    if opt.get("bg"):
        kw["background"] = torch.rand(n, 3, generator=g).to(dev)
    if opt.get("white"):
        kw["white_bkgd"] = True
    out = eng.render(ro.to(dev), rd.to(dev), 0.2, 0.8, nc, nf, **kw)
    torch.cuda.synchronize()
    return {k: _digest(v) for k, v in sorted(out.items()) if isinstance(v, torch.Tensor)}


def chunked_train_digests(dev, eng, prec):
    """The training forward over 200 rays at 64c+64f in chunks of 32 rays (the last one ragged)."""
    n, nc, nf = 200, 64, 64
    fr, ro, rd = _rays(n, 9)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    g = torch.Generator().manual_seed(17)
    noise = {"t_rand": torch.rand(n, nc, generator=g).to(dev), "n_c": torch.randn(n, nc, generator=g).to(dev),
             "u": torch.rand(n, nf, generator=g).to(dev), "n_f": torch.randn(n, nc + nf, generator=g).to(dev)}
    bg = torch.rand(n, 3, generator=g).to(dev)
    os.environ["NFB_TRAIN_MEM_MB"] = "48"  # read by the library on every call
    try:
        out = eng.render(ro.to(dev), rd.to(dev), 0.2, 0.8, nc, nf, perturb=True, noise_std=1.0, background=bg, noise=noise,
                         precision=prec, train=True)
        torch.cuda.synchronize()
    finally:
        del os.environ["NFB_TRAIN_MEM_MB"]
    return {k: _digest(v) for k, v in sorted(out.items()) if isinstance(v, torch.Tensor)}


def all_digests(dev):
    eng = _engine(dev)
    res = {}
    for prec in ("fast", "exact"):
        for name in CASES:
            res[f"{prec}/{name}"] = case_digests(dev, eng, name, prec)
        res[f"{prec}/chunked_train_64c64f"] = chunked_train_digests(dev, eng, prec)
    return res


@pytest.fixture(scope="module")
def dev(built_lib):
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng(dev):
    return _engine(dev)


@pytest.fixture(scope="module")
def stored():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.mark.parametrize("prec", ["fast", "exact"])
@pytest.mark.parametrize("name", list(CASES))
def test_case_equals_the_stored_run(dev, eng, stored, name, prec):
    got = case_digests(dev, eng, name, prec)
    want = stored[f"{prec}/{name}"]
    assert got == want, [k for k in want if got.get(k) != want[k]]


@pytest.mark.parametrize("prec", ["fast", "exact"])
def test_chunked_training_forward_equals_the_stored_run(dev, eng, stored, prec):
    got = chunked_train_digests(dev, eng, prec)
    want = stored[f"{prec}/chunked_train_64c64f"]
    assert got == want, [k for k in want if got.get(k) != want[k]]


if __name__ == "__main__":
    print(json.dumps(all_digests(torch.device("cuda", 0)), indent=1, sort_keys=True))
