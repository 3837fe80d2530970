"""The small tensor helpers of the drop-in `nerf` package (nerf/nerf_helpers.py) that the reference's unmodified scripts call on
the host side of the boundary, against what the reference's own functions return on CPU: same values bit for bit, same shapes,
same chunking.  The reference's results on these inputs were recorded by running it (oracle/make_golden_live.py ->
tests/golden/live/dropin_helpers.npz); CPU only."""
import os

import numpy as np
import pytest
import torch

import golden_io
import make_golden_live as ML
import nerface_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "dropin_helpers.npz")


@pytest.fixture(scope="module")
def both(built_lib):
    import nerf
    return nerf, golden_io.load(GOLD)


@pytest.mark.parametrize("H,W,intr", ML.RAY_BUNDLE_CASES)
def test_get_ray_bundle(both, H, W, intr):
    nerf, gold = both
    pose = ML.dropin_pose(H * 100 + W)
    want = gold["ray_bundle"][ML.RAY_BUNDLE_CASES.index((H, W, intr))]
    got = nerf.get_ray_bundle(H, W, intr, pose)
    got34 = nerf.get_ray_bundle(H, W, np.array(intr), pose[:3, :4])
    for a, b, c in zip(want, got, got34):
        assert a.shape == b.shape == (H, W, 3) and torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("n_freq,include_input,log_sampling", ML.PE_CASES)
def test_positional_encoding_and_embedding_function(both, n_freq, include_input, log_sampling):
    nerf, gold = both
    k = ML.PE_CASES.index((n_freq, include_input, log_sampling))
    x = torch.randn(37, 3, generator=torch.Generator().manual_seed(n_freq)) * 3.0
    want = gold["pe"][k]
    got = nerf.positional_encoding(x, n_freq, include_input, log_sampling)
    assert want.shape == got.shape and torch.equal(want, got)
    f = nerf.get_embedding_function(n_freq, include_input, log_sampling)
    assert torch.equal(gold["embedding"][k], f(x))


def test_meshgrid_minibatches_and_metrics(both):
    nerf, gold = both
    a, b = torch.arange(5, dtype=torch.float32), torch.arange(3, dtype=torch.float32) * 2.0
    got = nerf.meshgrid_xy(a, b)
    assert len(got) == len(gold["meshgrid"])
    for u, v in zip(gold["meshgrid"], got):
        assert u.shape == v.shape and torch.equal(u, v)
    x = torch.randn(23, 4, generator=torch.Generator().manual_seed(3))
    for w, cs in zip(gold["minibatches"], (1, 7, 23, 100)):
        g = nerf.get_minibatches(x, chunksize=cs)
        assert len(w) == len(g) and all(torch.equal(p, q) for p, q in zip(w, g))
    y = torch.randn(23, 4, generator=torch.Generator().manual_seed(4))
    assert torch.equal(gold["img2mse"], nerf.img2mse(x, y))
    for want, m in zip(gold["mse2psnr"], (0.0, 1e-5, 0.0123, 1.0)):
        got = nerf.mse2psnr(m)
        assert type(got) is type(want) and got == want


def test_cfgnode_on_a_script_shaped_config(both):
    """The scripts build `CfgNode(yaml.load(...))`, read nested attributes and write `cfg.dump()` next to the checkpoints
    (train_transformed_rays.py:46-50, 126-128): same tree, same leaves and leaf types as the reference's CfgNode on the same
    config, a dump that loads back to the same dict."""
    import yaml
    nerf, gold = both
    b = nerf.CfgNode(ML.CFG_RAW)

    def leaves(node, trail):
        res = []
        for k in node.keys():
            v = getattr(node, k)
            if isinstance(v, dict):
                assert isinstance(v, nerf.CfgNode), trail + [k]
                res.append([trail + [k], "dict", "CfgNode"])
                res += leaves(v, trail + [k])
            else:
                res.append([trail + [k], type(v).__name__, v])
        return res

    key = lambda e: tuple(e[0])  # noqa: E731
    assert sorted(leaves(b, []), key=key) == sorted(gold["cfg_leaves"], key=key)
    assert b.nerf.train.num_coarse == 64 and b.nerf.validation.num_fine == 64 and b.dataset.no_ndc is True
    assert gold["cfg_dump_roundtrip_equal"] and yaml.safe_load(b.dump()) == ML.CFG_RAW
    with pytest.raises(AttributeError):
        b.nerf.no_such_option


def test_model_class_against_the_reference_class(both):
    """ConditionalBlendshapePaperNeRFModel built with the keyword arguments the scripts pass (train_transformed_rays.py:150-176):
    same state_dict keys / shapes / dtypes and parameter count as the reference class, the same parameters load strictly, the
    torch forward of the drop-in (not the hot path) returns the reference module's values bit for bit, and the attributes the
    scripts and the renderer read are the same."""
    nerf, gold = both
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(**ML.MODEL_KW)
    sd = m.state_dict()
    assert [[k, list(v.shape), str(v.dtype)] for k, v in sd.items()] == gold["state_dict"]
    m.load_state_dict(O.random_init_params(100), strict=True)
    for name, want in gold["attributes"].items():
        assert getattr(m, name) == want, name
    g = torch.Generator().manual_seed(12)
    x = torch.randn(19, m.dim_xyz + m.dim_dir, generator=g)
    expr, lat = torch.randn(76, generator=g), torch.randn(32, generator=g)
    with torch.no_grad():
        assert torch.equal(m(x, expr, lat), gold["forward"])
    assert sum(p.numel() for p in m.parameters()) == gold["numel"]
