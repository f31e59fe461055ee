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


TEAMS = (1, 3, 8)


def team_params(cases, big_rows=2000):
    """pytest params (case, team) running every case of kernel 13's builders at each team size of TEAMS: the team of one
    with the ids the cases had before teams, the others as "<case>-team<t>"; cases of big_rows rows or more at teams 1
    and 3 only (a team of 8 host threads meets its barrier thousands of times per node).  A case is (name, X, ...)."""
    out = []
    for c in cases:
        for t in TEAMS:
            if t == 1 or t == 3 or c[1].shape[0] < big_rows:
                out.append(pytest.param(c, t, id=c[0] if t == 1 else "%s-team%d" % (c[0], t)))
    return out


def tsan_flags():
    """nvcc flags of a ThreadSanitizer build of a host harness, or skip the test when the toolchain has no libtsan."""
    res = subprocess.run(["gcc", "-print-file-name=libtsan.so"], capture_output=True, text=True) if shutil.which("gcc") else None
    if res is None or res.returncode != 0 or not os.path.isabs(res.stdout.strip()):
        pytest.skip("libtsan not available")
    return ("-g", "-Xcompiler", "-fsanitize=thread", "-Xlinker", "-ltsan")


def tsan_reports(cmd, log_prefix, timeout=120):
    """Run a ThreadSanitizer build of a harness (``cmd``) with its reports logged to ``log_prefix``.<pid>, and return them.

    Meant for builds with a barrier deleted: such a build reads what another thread has not written yet, and what it
    does next (a wrong tree, an index past a buffer, a crash, a loop that does not end) depends on timing.  So its exit
    status and output are ignored and it is killed after ``timeout`` seconds; only the race reports count, and
    ThreadSanitizer writes those at the racing access, before anything that access leads to."""
    env = dict(os.environ, TSAN_OPTIONS="exitcode=0 log_path=%s" % log_prefix)
    try:
        subprocess.run(cmd, capture_output=True, timeout=timeout, env=env)
    except subprocess.TimeoutExpired:
        pass
    d, base = os.path.split(str(log_prefix))
    return "".join(open(os.path.join(d, f), errors="replace").read() for f in sorted(os.listdir(d)) if f.startswith(base + "."))


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
