"""The oracle against the UNMODIFIED reference (CPU), on configurations the golden fixtures of tests/test_oracle_golden.py do not
hold: the smallest sample counts the kernels accept, a single fine sample, ragged chunk sizes, perturbation without noise, white
background without a background image, the direction-ablation input with every stochastic option on.  Every output must be
bit-identical.  What the reference returned, and the random tensors it drew in its own order, were recorded by running it on
these inputs (oracle/make_golden_live.py -> tests/golden/live/oracle_cases.npz).  CPU only."""
import os

import pytest
import torch

import golden_io
import make_golden_live as ML
import nerface_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "oracle_cases.npz")
CASES = ML.ORACLE_CASES


@pytest.fixture(scope="module")
def gold():
    assert torch.get_float32_matmul_precision() == "highest"
    return golden_io.load(GOLD)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_is_bit_identical_to_the_live_reference(gold, name):
    H, W, s, mode, use_bg, use_fine, stress, ablation = CASES[name]
    ci, pc, pf, fr, fr2 = ML.oracle_case_inputs(name)
    g = gold[name]
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    assert torch.equal(g["ray_bundle"][0], ro) and torch.equal(g["ray_bundle"][1], rd)
    if mode == "train":  # the trainer passes flat gathered rays (train_transformed_rays.py:320-326)
        ro, rd = ro.reshape(-1, 3).clone(), rd.reshape(-1, 3).clone()
    bg = fr["bg"].reshape(-1, 3) if use_bg else None
    rd_abl = None
    if ablation:
        rd_abl = O.ray_bundle(H, W, fr2["intrinsics"], fr2["pose"])[1]
        assert torch.equal(g["rd_ablation"], rd_abl)
    want = g["want"]
    # the recorded draws, split back into the per-chunk order the reference made them in (train_utils.py:69-76, 105-119)
    n_rays = H * W
    it = iter(g["draws"])
    noises = []
    for st in range(0, n_rays, s.chunksize):
        nz = O.Noise()
        if s.perturb:
            nz.t_rand = next(it)
        if s.noise_std > 0:
            nz.n_c = next(it)
        if s.num_fine > 0:
            if s.perturb:
                nz.u = next(it)
            if s.noise_std > 0:
                nz.n_f = next(it)
        noises.append(nz)
    assert next(it, None) is None, "the reference drew more random tensors than the oracle's model of it consumes"
    with torch.no_grad():
        got = O.run_one_iter(ro, rd, pc, pf, s, ML.NEAR, ML.FAR, fr["expr"], fr["latent"], bg, mode, noise_per_chunk=noises,
                             rd_ablation=rd_abl)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(want, got)):
        assert (a is None) == (b is None), i
        if a is not None:
            assert a.shape == b.shape, (i, a.shape, b.shape)
            assert torch.equal(a, b), (name, i, float((a - b).abs().max()))
