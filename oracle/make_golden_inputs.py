"""Generate tests/golden/live/backward_inputs.npz: the UNMODIFIED reference's autograd gradients with respect to the render's
inputs, for tests/test_input_grads_reference_cpu.py.

The training loss of train_transformed_rays.py:355-389 (mse of the coarse and the fine colour against the target) is
back-propagated through the live reference's run_one_iter_of_nerf in mode "train", with perturbation and sigma noise on, and
with ray_origins, ray_directions, expressions, background_prior and latent_code as leaves that require grad.  The cases are
the three of backward.npz (make_golden_live.BACKWARD_CASES, same inputs) plus "ablation": ray_directions_ablation also
requires grad, and the batch is split into two chunks of 5 rays, so the reference's direction encoder reads chunk 0 of the
ablation bundle in both chunks (train_utils.py:81-82).  Stored: outputs, the random draws, the loss and every input gradient
(the tensors are small).  Kept in its own file so that regenerating it leaves the other golden files untouched.

Usage:  python oracle/make_golden_inputs.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import golden_io  # noqa: E402
import make_golden_live as ML  # noqa: E402
import nerface_oracle as O  # noqa: E402

# tag: (stress, white, use_bg, ablation, chunksize)
INPUT_CASES = {**{tag: (*v, False, 2048) for tag, v in ML.BACKWARD_CASES.items()}, "ablation": (False, False, True, True, 5)}


def ablation_bundle(H, W):
    fr2 = O.synthetic_frame(32, H, W)
    return O.ray_bundle(H, W, fr2["intrinsics"], fr2["pose"])[1].reshape(-1, 3).clone()


def gen_backward_inputs(ref, rl):
    import make_golden as MG
    out = {}
    orig_relu = torch.nn.functional.relu
    torch.nn.functional.relu = lambda x, *a, **k: orig_relu(x).clone()  # the gradient-baseline patch (ref_loader docstring)
    try:
        for tag, (stress, white, use_bg, ablation, chunk) in INPUT_CASES.items():
            H, W, s, fr, pc, pf, ro, rd, bg, target = ML.backward_inputs(stress, white, use_bg)
            mc, mf = rl.build_model(ref, pc), rl.build_model(ref, pf)
            leaves = {"ray_origins": ro.clone(), "ray_directions": rd.clone(), "expressions": fr["expr"].clone(),
                      "latent_code": fr["latent"].clone()}
            if bg is not None:
                leaves["background_prior"] = bg.clone()
            if ablation:
                leaves["ray_directions_ablation"] = ablation_bundle(H, W)
            for t in leaves.values():
                t.requires_grad_(True)
            cfg = rl.make_cfg(ref, s.num_coarse, s.num_fine, True, 0.1, white, chunk, "train", ML.NEAR, ML.FAR)
            torch.manual_seed(77)
            with MG.Recorder() as rec:
                o = ref.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, leaves["ray_origins"], leaves["ray_directions"], cfg,
                                             mode="train", encode_position_fn=ref.get_embedding_function(10, True, True),
                                             encode_direction_fn=ref.get_embedding_function(4, False, True),
                                             expressions=leaves["expressions"], background_prior=leaves.get("background_prior"),
                                             latent_code=leaves["latent_code"],
                                             ray_directions_ablation=leaves.get("ray_directions_ablation"))
            loss = torch.nn.functional.mse_loss(o[0][..., :3], target) + torch.nn.functional.mse_loss(o[3][..., :3], target)
            loss.backward()
            out[tag] = {"out": [t.detach() for t in o], "draws": [t for _, t in rec.draws], "loss": float(loss.detach()),
                        "chunksize": chunk, "inputs": {k: v.detach().clone() for k, v in leaves.items()},
                        "grads": {k: v.grad.clone() for k, v in leaves.items()}}
    finally:
        torch.nn.functional.relu = orig_relu
    return out


def main():
    import ref_loader as rl
    assert torch.get_float32_matmul_precision() == "highest"
    ref = rl.load_reference()
    assert ref is not None, "no reference tree"
    golden_io.save(os.path.join(ML.GOLDEN, "backward_inputs.npz"), gen_backward_inputs(ref, rl))


if __name__ == "__main__":
    main()
