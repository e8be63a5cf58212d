"""Build the CUDA library in-tree for sm_90a (H100; nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "b200pde.cu")
import glob
DEPS = sorted(glob.glob(os.path.join(HERE, "csrc", "*"))) + [os.path.join(HERE, "..", "include", "b200pde.h")]
OUT = os.path.join(HERE, "libb200pde.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    tmp = f"{OUT}.{os.getpid()}.tmp"   # build aside and rename: a reader (another rank, a snapshot) never sees a half-written library
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-shared", "-Xcompiler", "-fPIC", "-o", tmp, SRC]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True)
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
