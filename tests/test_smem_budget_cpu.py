"""CPU: shared-memory budgets of the two feature kernels for the shapes the library instantiates, and of kernel 13's three
build kernels for every shape their launchers accept.

sm_90: 233 472 B of shared memory per SM, 1 024 B reserved per resident CTA, so n CTAs per SM need
n * (bytes + 1024) <= 233 472.  The CTA kernel (csrc/fast_kernel.cuh) is sized for 3 CTAs per SM on the headline shape;
the pair kernel (csrc/pair_kernel.cuh) runs one CTA of up to 20 autonomous warps per SM (9.6 KB of shared memory per warp on
the headline shape, five warps per scheduler at 96 registers).  The generic kernel (csrc/generic_kernel.cuh) takes 8, 4,
2 or 1 frames per CTA group by the same budget, or keeps its window-sized arrays in global scratch."""
import os
import re
import subprocess

from tests import host_exe
from tests.kernels import GENERIC_SWEEP

SM_BYTES, CTA_RESERVED = 233472, 1024


def ctas_per_sm(nbytes):
    return SM_BYTES // (nbytes + CTA_RESERVED)


def test_shared_memory_budget(tmp_path_factory):
    exe = host_exe.build(tmp_path_factory, "smem_budget_host.cu")
    windows = ["%d:%d" % (fs, w) for fs, w, _, _ in GENERIC_SWEEP]
    lines = [ln.split() for ln in subprocess.run([exe] + windows, capture_output=True, text=True).stdout.splitlines()]
    # the generic kernel's spectrum sweep reaches the group size (and transform form) each window is listed for, with the
    # tables blob its plan builds and with 256 words less or more: a change to the budget formula or to the tables' size
    # that moves a window across a threshold fails here instead of silently moving the sweep off its targets
    generic = {(int(l[1]), int(l[2])): [int(v) for v in l[3:]] for l in lines if l[0] == "generic"}
    assert len(generic) == len(GENERIC_SWEEP)
    for fs, w, G, what in GENERIC_SWEEP:
        Nc, words, g_less, g, g_more, nbytes = generic[(fs, w)]
        assert Nc == (w // 2 if w % 2 == 0 else w), (w, Nc)
        assert words > 700, (fs, w, words)          # mel taps + DCT + chroma of a real plan
        assert g_less == g == g_more == G, (fs, w, what, words, G, (g_less, g, g_more))
        # 8 frames per group: two CTAs per SM (the kernel's __launch_bounds__); any other group: one
        assert ctas_per_sm(nbytes) >= (2 if g == 8 else 1), (fs, w, g, nbytes)
    table = {(int(l[1]), int(l[2])): (int(l[3]), int(l[4])) for l in lines if l[0] == "fast"}
    assert len(table) == 15
    # headline shape (50 / 25 ms @ 16 kHz): 3 CTAs per SM
    runs, d = table[(800, 400)]
    assert runs == 1 and ctas_per_sm(d) == 3
    # every instantiated shape keeps at least 2 CTAs per SM at hop = window / 2 and fits the launcher's 110 KB cap
    for (n, s), (runs, d) in table.items():
        assert d <= 110 * 1024, (n, s, d)
        if 2 * s <= n:
            assert ctas_per_sm(d) >= 2, (n, s, d)
    pair = {int(l[1]): (int(l[2]), int(l[3])) for l in lines if l[0] == "pair"}
    assert set(pair) == {320, 480, 512, 640, 800, 960, 1024}
    for w, (warps, nbytes) in pair.items():
        assert ctas_per_sm(nbytes) >= 1 and nbytes <= 227 * 1024, (w, warps, nbytes)     # pair_launch_t's cap (kPairCtaCap)
        assert warps >= 16 and warps % 4 == 0, (w, warps)     # whole rounds over the four schedulers of an SM
    assert pair[800][0] == 20         # 20 autonomous warps per SM on the headline shape


# sm_90's largest opt-in dynamic shared memory per CTA (cudaDevAttrMaxSharedMemoryPerBlockOptin: 227 KB)
SM90_OPTIN = 227 * 1024


def test_kernel13_shared_memory_caps(tmp_path_factory):
    """Kernel 13's three build kernels: every accepted shape (F <= 512, C <= 32) fits under the kernel's cap, the cap is
    the size at the largest shape, every cap is below sm_90's opt-in maximum, at every accepted shape the carve of the
    shared memory (forest.cuh carve_smem / carve_reg_smem) ends within the size formula the launchers pass, and every
    cudaFuncSetAttribute in forest.cu passes a cap constant, with at least one per build kernel.  A launcher that set its
    own call's size instead would let a concurrent call of a smaller shape lower the limit between another thread's set
    and launch, and that launch would fail."""
    csrc = os.path.join(host_exe.ROOT, "pyaudioanalysis_b200", "csrc")
    exe = host_exe.build(tmp_path_factory, "forest_smem_host.cu", "-I" + csrc)
    lines = [ln.split() for ln in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()]
    caps = {ln[0]: (int(ln[1]), int(ln[2]), ln[3]) for ln in lines}
    assert set(caps) == {"forest_build_kernel", "forest_reg_build_kernel", "boost_build_kernel"}
    for kern, (cap, largest, shape) in caps.items():
        assert largest == cap, (kern, cap, largest, shape)
        assert cap <= SM90_OPTIN, (kern, cap)
    assert caps["forest_build_kernel"] == (49832, 49832, "512:32")          # past the 48 KB default
    past = {ln[0]: int(ln[4]) for ln in lines}
    assert past == dict.fromkeys(caps, 0), past
    src = open(os.path.join(csrc, "forest.cu")).read()
    calls = re.findall(r"cudaFuncSetAttribute\(\s*(\w+)\s*,\s*cudaFuncAttributeMaxDynamicSharedMemorySize\s*,\s*([^;]*?)\)\);", src)
    assert len(calls) == src.count("cudaFuncSetAttribute(") == 5, calls
    want = {"forest_build_kernel": "int(forest::kSmemCap)", "forest_reg_build_kernel": "int(forest::kRegSmemCap)",
            "boost_build_kernel": "int(forest::kBoostSmemCap)"}
    for kern, arg in calls:
        assert want[kern] == arg.strip(), (kern, arg)
    assert {kern for kern, _ in calls} == set(want), calls
