"""Compile libb200aa.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200aa.so")
HEADER = os.path.join(HERE, "..", "include", "b200aa.h")
SOURCES = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
DEPS = sorted(glob.glob(os.path.join(CSRC, "*"))) + [HEADER]

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-shared", "-Xcompiler", "-fPIC"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def compile_lib(out, extra_flags=(), verbose=False):
    """Compile every csrc/*.cu in one nvcc invocation into the shared library `out`; -v adds ptxas's per-kernel report."""
    cmd = [_nvcc()] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building " + os.path.basename(out))
    if verbose:
        sys.stderr.write(res.stderr)


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    """Build the library if it is missing or older than its sources.  Returns the path."""
    if not force and not needs_build():
        return LIB
    compile_lib(LIB + ".tmp", verbose=verbose)
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
