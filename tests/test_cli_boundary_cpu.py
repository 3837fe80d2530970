"""The reference's UNMODIFIED training script on the drop-in package, as far as a machine without a GPU can take it: through
4d-facial-avatars_b200/run_reference_script.py it imports `nerf` (ours), parses the shipped paper-model YAML, loads the synthetic
FLAME-style dataset with our loader, builds both networks, the latent codes and the optimizer, draws the first importance-sampled
ray batch — and stops exactly at its first `run_one_iter_of_nerf` call (train_transformed_rays.py:336), where the product path
refuses to run without CUDA (no CPU fallback).  On an H100 the same command trains.  Needs the reference tree."""
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_loader  # noqa: E402

pytestmark = [pytest.mark.skipif(ref_loader.reference_root() is None, reason="no reference tree (run oracle/stage_reference.py)"),
              pytest.mark.skipif(torch.cuda.is_available(), reason="with a GPU the script trains: tools/run_reference_clis.py")]


def test_unmodified_train_script_reaches_the_boundary(tmp_path, built_lib):
    out = str(tmp_path)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_reference_clis.py"), "--out", out, "--gpus", "1",
                          "--iters", "4", "--size", "64", "--test-frames", "6"], capture_output=True, text=True, timeout=600, cwd=out)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]   # the driver reports; the script's own rc is in the summary
    log = open(os.path.join(out, "train_g1.log")).read()
    assert "there is no CPU fallback" in log
    # the traceback passes through the script's own call of run_one_iter_of_nerf (unmodified file, reference tree)
    frames = re.findall(r'File "([^"]+)", line (\d+), in (\w+)', log)
    script = [f for f in frames if f[0].endswith("train_transformed_rays.py")]
    assert script and script[-1][2] == "main" and 330 <= int(script[-1][1]) <= 352, script
    assert os.path.realpath(script[-1][0]).startswith(os.path.realpath(ref_loader.reference_root()))
    ours = [f for f in frames if os.sep + "4d-facial-avatars_b200" + os.sep + "nerf" + os.sep in f[0]]
    assert ours and ours[0][2] == "run_one_iter_of_nerf"
    assert '"rc": 1' in res.stdout and '"checkpoint": false' in res.stdout


def test_unmodified_eval_script_reaches_the_boundary(tmp_path, built_lib):
    """Same for eval_transformed_rays.py with a checkpoint in the train script's format (train_transformed_rays.py:555-566): it
    loads both state_dicts into the drop-in model class, the background and the latent codes, builds the test-set loop and stops
    at its first run_one_iter_of_nerf call (eval_transformed_rays.py:449-467)."""
    import nerface_oracle as O
    out = str(tmp_path)
    # dataset + YAML exactly as the driver of the GPU runs prepares them (the train attempt itself ends at the boundary, above);
    # 244 test frames: the unedited eval loop reads pose 100 and the direction bundle of frame 240 + i (SURVEY.md §8b)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_reference_clis.py"), "--out", out, "--gpus", "1",
                          "--iters", "4", "--size", "64", "--test-frames", "244"], capture_output=True, text=True, timeout=600, cwd=out)
    assert res.returncode == 0
    ckpt = os.path.join(out, "synthetic.ckpt")
    torch.save({"iter": 3, "model_coarse_state_dict": O.random_init_params(100), "model_fine_state_dict": O.random_init_params(101),
                "optimizer_state_dict": None, "loss": 0.1, "psnr": 10.0, "background": torch.zeros(64, 64, 3),
                "latent_codes": torch.zeros(12, 32)}, ckpt)
    launcher = os.path.join(ROOT, "4d-facial-avatars_b200", "run_reference_script.py")
    ev = subprocess.run([sys.executable, launcher, ref_loader.script_path("eval_transformed_rays.py"), "--config",
                         os.path.join(out, "synthetic_g1.yml"), "--checkpoint", ckpt, "--savedir", os.path.join(out, "renders")],
                        capture_output=True, text=True, timeout=600, cwd=out, env=dict(os.environ, MPLBACKEND="Agg"))
    log = ev.stdout + ev.stderr
    assert ev.returncode != 0 and "there is no CPU fallback" in log, log[-3000:]
    assert "loaded latent codes from checkpoint" in log and "loaded background with shape" in log
    frames = re.findall(r'File "([^"]+)", line (\d+), in (\w+)', log)
    script = [f for f in frames if f[0].endswith("eval_transformed_rays.py")]
    assert script and 440 <= int(script[-1][1]) <= 470, script
    assert os.path.realpath(script[-1][0]).startswith(os.path.realpath(ref_loader.reference_root()))
