"""Build the CUDA engine in-tree:  python-paillier_b200/libpaillier_b200.so  (sm_90a only).

nvcc cross-compiles without a GPU.  The .so is git-ignored but travels to the GPU box with the
repo snapshot.  Rebuilds only when a source or this file is newer than the library.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpaillier_b200.so")
SOURCES = ["pai_engine.cu"]
HEADERS = ["pai_core.cuh", "pai_kernels.cuh", "pai_digit.cuh", "pai_cta.cuh", "pai_coop.cuh", "pai_tc.cuh", "pai_rng.cuh", "pai_radix.cuh", "pai_pack.cuh", "pai_rt.h", os.path.join("..", "..", "include", "paillier_b200.h")]
# --split-compile 0: the device optimisation of the many kernel instantiations runs on every host core
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--split-compile", "0",
              "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v"]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    """True when the library is missing or older than a source or than this file (which holds the flags and the target
    architecture)."""
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = [find_nvcc()] + NVCC_FLAGS + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log[-4000:])
        raise RuntimeError("nvcc failed (see %s/build.log)" % HERE)
    if verbose:
        print(log[-2000:])
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
