"""nerf.parallel.data_parallel all-reduces parameter and latent gradients only: when an input of run_one_iter_of_nerf that it
would have to reduce requires grad, it refuses instead of returning per-shard partial gradients (no GPU needed)."""
import pytest
import torch


@pytest.mark.parametrize("which", ["ray_origins", "ray_directions", "expressions", "background_prior", "ray_directions_ablation"])
def test_data_parallel_refuses_input_gradients(monkeypatch, which):
    from nerf import parallel
    monkeypatch.setattr(parallel.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(parallel.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(parallel.dist, "get_rank", lambda group=None: 0)
    called = []
    wrapped = parallel.data_parallel(lambda *a, **k: called.append(1))
    n = 8
    kw = dict(ray_origins=torch.zeros(n, 3), ray_directions=torch.ones(n, 3), expressions=torch.zeros(76),
              background_prior=torch.zeros(n, 3), ray_directions_ablation=torch.ones(n, 3))
    kw[which].requires_grad_(True)
    with pytest.raises(NotImplementedError, match="data_parallel"):
        wrapped(2, 4, 10.0, None, None, kw["ray_origins"], kw["ray_directions"], None, mode="train", expressions=kw["expressions"],
                background_prior=kw["background_prior"], latent_code=torch.zeros(32, requires_grad=True),
                ray_directions_ablation=kw["ray_directions_ablation"])
    assert not called
