"""Stage the UNMODIFIED reference files of the hot path into `oracle/_ref/` (test / baseline infrastructure, not product).

The recipe copies — byte for byte, nothing edited — the reference's `nerf` package, the two CLI scripts that call the
path and the shipped paper-model YAML from a reference checkout into `oracle/_ref/` (git-ignored: reference sources never
enter this repository).  It is the offline "install" of a reference that has no setup.py, so a machine that has the built
tree but not the reference checkout can still run it.  Users of the staged copy:

  * bench.py --impl reference and the `cpu_baseline` / `gpu_baseline` legs (`kind: "reference"`): the reference's own
    run_one_iter_of_nerf on the host cores / on the GPU through torch CUDA with TF32 off (the oracle port when nothing is staged);
  * tests/test_cli_boundary_cpu.py and run_reference_script.py: the unmodified train_transformed_rays.py /
    eval_transformed_rays.py with this repo's drop-in `nerf` package first on sys.path;
  * oracle/make_golden_live.py --cuda: the eval script's post-render functions on torch CUDA.

    python oracle/stage_reference.py [--ref /root/reference]

`__graft_entry__.build()` runs it whenever the reference checkout is readable.
"""
import argparse
import hashlib
import json
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEST = os.path.join(ROOT, "oracle", "_ref")
NP = os.path.join("nerface_code", "nerf-pytorch")
FILES = [os.path.join(NP, "nerf", f) for f in (
    "__init__.py", "cfgnode.py", "load_blender.py", "load_flame.py", "load_llff.py", "models.py", "nerf_helpers.py",
    "train_utils.py", "volume_rendering_utils.py")] + [
    os.path.join(NP, "train_transformed_rays.py"), os.path.join(NP, "eval_transformed_rays.py"),
    os.path.join(NP, "config", "dave", "dave_dvp_lcode_fixed_bg_512_paper_model.yml")]


def stage(ref_root="/root/reference", dest=DEST):
    """Copy FILES from ref_root to dest (same relative paths) + MANIFEST.json with their sha256.  Returns dest, or None
    when the reference tree is absent or unreadable (an earlier staged copy is then used as is)."""
    if not all(os.access(os.path.join(ref_root, rel), os.R_OK) for rel in FILES):
        return None
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(ref_root, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        with open(dst, "rb") as f:
            manifest[rel] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, "MANIFEST.json"), "w") as f:
        json.dump({"source": ref_root, "files": manifest}, f, indent=1)
    return dest


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    d = stage(a.ref)
    print(d if d else f"{a.ref} not found: nothing staged")
