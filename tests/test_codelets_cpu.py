"""CPU: the register FFT codelets of the fused kernel (csrc/dft_codelets.cuh are __host__ __device__ templates) and the
R1 x R2 packed-real transform built from them, run on the host against a naive float64 DFT (tests/codelets_host.cu)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_codelets_and_shapes_on_host(tmp_path):
    exe = str(tmp_path / "codelets_host")
    res = subprocess.run([_nvcc(), "-std=c++17", "-O1", "-arch=sm_90a", "-o", exe, os.path.join(ROOT, "tests", "codelets_host.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0, run.stdout
    lines = [ln.split() for ln in run.stdout.splitlines()]
    codelets = {int(l[1]) for l in lines if l[0] == "codelet"}
    shapes = {(int(l[1]), int(l[2])) for l in lines if l[0] == "shape"}
    assert codelets == {10, 12, 15, 16, 20, 21, 25, 30, 32}
    assert {int(l[1]) for l in lines if l[0] == "pair"} == {10, 15, 20, 25, 30}     # pair_r_for_window in csrc/pair_kernel.cuh
    # every (R1, R2) the library instantiates (fast_shape_for_window in csrc/fast_kernel.cuh, solo_shape_for_window in
    # csrc/solo_kernel.cuh as (R2, L))
    assert shapes == {(20, 20), (21, 21), (20, 10), (20, 12), (20, 15), (16, 10), (20, 16), (10, 20), (15, 20)}
    assert all(float(l[3]) < 2e-6 for l in lines if l[0] in ("codelet", "shape", "pair", "soa32"))
