"""Host harnesses of the CPU tests: a C++ source that includes csrc/ headers, compiled by nvcc for the host, so that the
__host__ __device__ pieces of the kernels (and the launchers' size rules) run on the CPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def nvcc():
    """Path of nvcc ($NVCC, the default CUDA install, or PATH), or None."""
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def build(tmp_path_factory, source, *flags):
    """Compile `source` (a file name under tests/, or an absolute path) with `nvcc -std=c++17 -arch=sm_90a` and `flags`
    into a fresh temporary directory and return the executable's path.  Skips the test when nvcc is missing."""
    if nvcc() is None:
        pytest.skip("nvcc not available")
    src = source if os.path.isabs(source) else os.path.join(ROOT, "tests", source)
    name = os.path.splitext(os.path.basename(src))[0]
    exe = str(tmp_path_factory.mktemp(name) / name)
    res = subprocess.run([nvcc(), "-std=c++17", *flags, "-arch=sm_90a", "-o", exe, src], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return exe
