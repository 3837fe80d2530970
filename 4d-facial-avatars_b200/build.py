"""Build lib/libnfb.so (the C-ABI shared library of include/nfb.h) in-tree with nvcc for sm_90a (H100).

The .so is git-ignored; rebuilds only when a source is newer than the library.  Usage: python 4d-facial-avatars_b200/build.py [--force] [--verbose] [--timers] | --variant NAME -D... (experiment build lib/libnfb_NAME.so)

--timers additionally builds lib/libnfb_timers.so with the phase timers compiled in (-DNFB_TIMERS=1; they cost registers in
the kernels' hot loops, so the product library does not carry them); tools/phase_profile.py loads it through NFB_LIB.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libnfb.so")
SOURCES = ["nfb_api.cu", "nfb_pack.cu", "nfb_optim.cu", "nfb_post.cu", "nfb_render.cu", "nfb_train.cu"]
HEADERS = ["nfb_internal.h", "nfb_layout.h", "nfb_pipeline.cuh", "nfb_ptx.cuh", "nfb_save.cuh", "nfb_render_common.cuh", "nfb_sampler.h", os.path.join("..", "..", "include", "nfb.h")]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, timers=False, variant=None, defines=()):
    """variant + defines: an experiment build lib/libnfb_<variant>.so with extra -D flags (select it with NFB_LIB)."""
    out = os.path.join(LIB_DIR, "libnfb_timers.so") if timers else LIB
    if variant:
        out = os.path.join(LIB_DIR, f"libnfb_{variant}.so")
    if not timers and not variant and not force and not needs_build():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in SOURCES if os.path.exists(os.path.join(CSRC, f))]
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
           "-Xcompiler", "-fPIC", "-shared", "-DNFB_BUILD"] + (["-DNFB_TIMERS=1"] if timers else []) + list(defines) + ["-o", out] + srcs
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building " + os.path.basename(out))
    if verbose:
        print(res.stdout + res.stderr)
    return out


if __name__ == "__main__":
    if "--variant" in sys.argv:  # python build.py --variant NAME -DFOO=1 [-DBAR=2 ...] [--timers]
        name = sys.argv[sys.argv.index("--variant") + 1]
        print(build(verbose="--verbose" in sys.argv, timers=False, variant=name, defines=[a for a in sys.argv if a.startswith("-D")]))
        sys.exit(0)
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
    if "--timers" in sys.argv:
        print(build(verbose="--verbose" in sys.argv, timers=True))
