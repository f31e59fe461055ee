"""Compile libb200aa.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200aa.so")
SOURCES = ["b200aa.cu"]
DEPS = ["b200aa.cu", "beat.cuh", "common.cuh", "dft_codelets.cuh", "generic_kernel.cuh", "fast_kernel.cuh", "knn.cuh", "pair_kernel.cuh", "pcm.cuh", "solo_kernel.cuh", "rows.cuh", "sched.cuh", "slots.h", "tables.inl",
        os.path.join("..", "..", "include", "b200aa.h")]

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-shared", "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force=False, verbose=False):
    """Build the library if it is missing or older than its sources.  Returns the path."""
    if not force and not needs_build():
        return LIB
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", LIB + ".tmp"] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libb200aa.so")
    if verbose:
        sys.stderr.write(res.stderr)
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
