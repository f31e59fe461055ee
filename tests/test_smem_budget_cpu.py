"""CPU: shared-memory budgets of the two feature kernels for the shapes the library instantiates.

sm_90: 233 472 B of shared memory per SM, 1 024 B reserved per resident CTA, so n CTAs per SM need
n * (bytes + 1024) <= 233 472.  The CTA kernel (csrc/fast_kernel.cuh) is sized for 3 CTAs per SM on the headline shape;
the pair kernel (csrc/pair_kernel.cuh) runs one CTA of up to 20 autonomous warps per SM (9.6 KB of shared memory per warp on
the headline shape, five warps per scheduler at 96 registers).  The generic kernel (csrc/generic_kernel.cuh) takes 8, 4,
2 or 1 frames per CTA group by the same budget, or keeps its window-sized arrays in global scratch."""
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
