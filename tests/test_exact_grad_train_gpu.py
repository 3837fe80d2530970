"""Exact-grad mode (NFB_PREC_EXACT_GRAD) through the fused trainer: eager and captured steps, one image and several images per
step, repeat an eager run bit for bit, as test_train_loop_gpu.py pins for the other two modes (same trainers, batches and
comparison)."""
import pytest
import torch

from test_train_loop_gpu import (E, env, assert_same_run, images_batches, one_image_batches, run_step, trainer,  # noqa: F401
                                 training_set, N_RAYS, ROUNDS)

pytestmark = pytest.mark.gpu


def test_eager_and_captured_steps_repeat_an_eager_run(E):
    """10 steps: graph only (K = 1), alternating eager / graph, and K = 4 x 512 image steps eager and captured, each against
    an eager-only trainer fed the same rays, after every step."""
    data, frs, images, single = training_set(E, n_images=4)
    batches = one_image_batches(E, data, frs, images, single, 10, seed=4)
    bks = images_batches(E, data, 4, 512, 10, seed=7)
    lat0 = torch.randn(4, 32, generator=torch.Generator().manual_seed(2)) * 0.1
    ref, ref_k = trainer(E, lat0, "exact_grad"), trainer(E, lat0, "exact_grad")
    runs = {"graph": "G" * 10, "alternating": "EGGEGEGGEE"}
    ts = {name: trainer(E, lat0, "exact_grad") for name in runs}
    tk = trainer(E, lat0, "exact_grad")
    tk.capture_images(data, 4, 512, max_rounds=ROUNDS, device_draws=False)
    for t in ts.values():
        t.capture(N_RAYS)
    for i, (b, bk) in enumerate(zip(batches, bks)):
        loss_ref = run_step(E, ref, "E", data, b, None, None)
        losses = {name: run_step(E, t, runs[name][i], data, b, None, None) for name, t in ts.items()}
        loss_k_ref = run_step(E, ref_k, "M", data, None, bk, 512)
        loss_k = run_step(E, tk, "IK" if i % 2 == 0 else "M", data, None, bk, 512)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss_ref).all())
        for name, t in ts.items():
            assert_same_run(E, ref, t, loss_ref, losses[name], f"exact_grad {name} step {i + 1} ({runs[name][i]})")
        assert_same_run(E, ref_k, tk, loss_k_ref, loss_k, f"exact_grad K=4 step {i + 1}")


def test_exact_grad_steps_leave_exact_steps_alone(E):
    """An exact-grad trainer on the same device first: exact-mode steps afterwards still repeat an exact-mode run on a device that
    never ran exact-grad (its forward, backward and re-pack are exact mode's, the lo stream only rides along)."""
    data, frs, images, single = training_set(E)
    batches = one_image_batches(E, data, frs, images, single, 3, seed=9)
    lat0 = torch.randn(3, 32, generator=torch.Generator().manual_seed(5)) * 0.1
    a = trainer(E, lat0, "exact")
    la = [run_step(E, a, "E", data, b, None, None) for b in batches]
    g = trainer(E, lat0, "exact_grad")
    lg = [run_step(E, g, "E", data, b, None, None) for b in batches]
    b2 = trainer(E, lat0, "exact")
    lb = [run_step(E, b2, "E", data, b, None, None) for b in batches]
    torch.cuda.synchronize()
    for x, y in zip(la, lb):
        assert torch.equal(x, y)
    assert torch.equal(a.params, b2.params)
    # the forward is exact mode's: the first step's loss is the same bits; the gradients (and so later steps) are not
    assert torch.equal(la[0], lg[0])
    assert not torch.equal(a.params, g.params)
