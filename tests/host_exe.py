"""Host harnesses of the CPU tests: a C++ source that includes csrc/ headers, compiled by nvcc for the host, so that the
__host__ __device__ pieces of the kernels (and the launchers' size rules) run on the CPU.

The stdin harnesses share one protocol (tests/host_io.h): numbers travel as hex floats, "inf" and "nan" (``hexes``,
``floats``), one command per line in, one result per line out (``run``)."""
import os
import shutil
import subprocess

import numpy as np
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


def hexes(values):
    """values (any shape) as float64 hex floats separated by spaces."""
    return " ".join(float(x).hex() for x in np.asarray(values, dtype=np.float64).ravel())


def run(exe, script):
    """Feed ``script`` to the harness ``exe``; its output lines, split into tokens."""
    res = subprocess.run([exe], input=script, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return [ln.split() for ln in res.stdout.splitlines()]


def floats(tokens):
    """float64 array of hex-float tokens ("nan" for NaN)."""
    return np.array([float.fromhex(t) if t != "nan" else np.nan for t in tokens])


def bits(a):
    """float64 bit patterns, every NaN mapped to 0x7ff8000000000000."""
    a = np.asarray(a, dtype=np.float64)
    b = a.view(np.uint64).copy()
    b[np.isnan(a)] = 0x7ff8000000000000
    return b
