"""The render kernel's schedule changes nothing it computes.

* The activation probe (`NfbDebug.act_dump`) runs in its own instantiation of `render_kernel`; the production
  instantiations carry no probe code.  The probe instantiation's outputs and per-sample dumps equal the production one's bit
  for bit, in both precision modes, so the tests that read the probe (test_render_fp64_gpu.py, test_parity_gpu.py) speak for
  the production kernel.
* Full frames (512², 64c+128f and 1024², 128c+256f in fast mode; 512² in exact mode) and a training forward (outputs,
  saved depths and colours, every byte of the activation records) equal a stored run of the kernel before the warpgroups
  ran their tiles independently (tests/golden/render_schedule_digests.json, SHA-256 of each array's bytes).

`python tests/test_render_schedule_gpu.py` prints the digests of the library it loads (NFB_LIB selects one) in the format of
that file.
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
DIGESTS = os.path.join(ROOT, "tests", "golden", "render_schedule_digests.json")
NAMES = ["rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last"]
FRAMES = {"fast_512_64c128f": ("fast", 512, 64, 128), "fast_1024_128c256f": ("fast", 1024, 128, 256),
          "exact_512_64c128f": ("exact", 512, 64, 128)}


def _engine_for_seeds(dev, seed_c=100, seed_f=101, stress=False):
    import nerf
    from nerf import _engine
    mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(), mk()
    mc.load_state_dict(O.random_init_params(seed_c, stress))
    mf.load_state_dict(O.random_init_params(seed_f, stress))
    eng = _engine.renderer_for(dev)
    eng.sync_weights(mc.to(dev), mf.to(dev))
    return eng


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def frame_digests(dev, key):
    prec, H, nc, nf = FRAMES[key]
    fr = O.synthetic_frame(1, H, H)
    eng = _engine_for_seeds(dev)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    bg = fr["bg"].reshape(-1, 3).to(dev).contiguous()
    v = eng.render_camera(fr["pose"], fr["intrinsics"], H, H, 0, H, 0.2, 0.8, nc, nf, background=bg, precision=prec)
    torch.cuda.synchronize()
    return {n: _digest(v[n]) for n in NAMES}


def train_digests(dev, prec):
    """The training forward (SAVE) with perturbation, noise and a background on 512 rays of the stress weights."""
    from test_backward_gpu import dev_tensor
    H = 32
    fr = O.synthetic_frame(5, H, 16)
    ro, rd = O.ray_bundle(H, 16, fr["intrinsics"], fr["pose"])
    n, nc, nf = H * 16, 64, 64
    g = torch.Generator().manual_seed(7)
    noise = {"t_rand": torch.rand(n, nc, generator=g), "n_c": torch.randn(n, nc, generator=g),
             "u": torch.rand(n, nf, generator=g), "n_f": torch.randn(n, nc + nf, generator=g)}
    eng = _engine_for_seeds(dev, 11, 12, stress=True)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    run = lambda: eng.render(ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev), 0.2, 0.8, nc, nf, perturb=True,  # noqa: E731
                             noise_std=1.0, background=fr["bg"].reshape(-1, 3).to(dev), noise=noise, precision=prec, train=True)
    # The record buffer belongs to the handle and holds bytes no record element covers (left from earlier calls): run once,
    # zero the buffer, and digest the records of a second run into the same buffer.
    run()
    torch.cuda.synchronize()
    d0 = eng.train_debug()
    dev_tensor(d0.records, (d0.n_tiles * d0.record_bytes // 4,), "<i4").zero_()
    out = run()
    torch.cuda.synchronize()
    d = eng.train_debug()
    assert d.records == d0.records and d.n_tiles == d0.n_tiles
    dg = {k: _digest(out[k]) for k in NAMES}
    dg["records"] = _digest(dev_tensor(d.records, (d.n_tiles, d.record_bytes // 4), "<i4"))
    dg["z_coarse"] = _digest(dev_tensor(d.z_coarse, (n, nc)))
    dg["raw_coarse"] = _digest(dev_tensor(d.raw_coarse, (n, nc, 4)))
    dg["z_fine"] = _digest(dev_tensor(d.z_fine, (n, nc + nf)))
    dg["raw_fine"] = _digest(dev_tensor(d.raw_fine, (n, nc + nf, 4)))
    dg["dnorm"] = _digest(dev_tensor(d.dnorm, (n,)))
    return dg


def all_digests(dev):
    res = {key: frame_digests(dev, key) for key in FRAMES}
    for prec in ("fast", "exact"):
        res[f"train_{prec}_512rays_64c64f"] = train_digests(dev, prec)
    return res


@pytest.fixture(scope="module")
def dev(built_lib):
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def stored():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.mark.parametrize("key", list(FRAMES))
def test_frame_equals_the_stored_run(dev, stored, key):
    assert frame_digests(dev, key) == stored[key]


@pytest.mark.parametrize("prec", ["fast", "exact"])
def test_training_forward_equals_the_stored_run(dev, stored, prec):
    got = train_digests(dev, prec)
    want = stored[f"train_{prec}_512rays_64c64f"]
    assert got == want, [k for k in want if got.get(k) != want[k]]


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("prec", ["fast", "exact"])
def test_probe_instantiation_equals_production(dev, prec):
    """Every output and per-sample dump (depths, raw MLP outputs of both passes) of a 128x128 frame on the stress weights,
    rendered by the production kernel and by the probe kernel at the PE dump (-1), the first and last layer and the
    direction layer (6)."""
    H, nc, nf = 128, 64, 128
    fr = O.synthetic_frame(2, H, H)
    ro, rd = O.ray_bundle(H, H, fr["intrinsics"], fr["pose"])
    eng = _engine_for_seeds(dev, 21, 22, stress=True)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    args = (ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev), 0.2, 0.8, nc, nf)
    kw = dict(background=fr["bg"].reshape(-1, 3).to(dev), precision=prec, debug=True)
    base = eng.render(*args, **kw)
    torch.cuda.synchronize()
    keys = NAMES + ["z_coarse", "raw_coarse", "z_fine", "raw_fine"]
    for step in (-1, 0, 6, 8):
        got = eng.render(*args, act_step=step, **kw)
        torch.cuda.synchronize()
        assert bool((got["act"] != 0).any()), f"the probe wrote nothing at step {step}"
        for k in keys:
            assert torch.equal(_bits(got[k]), _bits(base[k])), (prec, step, k)


if __name__ == "__main__":
    print(json.dumps(all_digests(torch.device("cuda", 0)), indent=1, sort_keys=True))
