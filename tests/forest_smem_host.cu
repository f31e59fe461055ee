// Host-side print of kernel 13's dynamic shared-memory sizes (pyaudioanalysis_b200/csrc/forest.cuh: smem_bytes,
// reg_smem_bytes, boost_smem_bytes) at every shape the launchers accept, F in 1 .. kMaxFeats and C in 1 .. kMaxClasses,
// against the caps the launchers set as the kernels' limits, and how many of those shapes the kernel's carve (carve_smem,
// carve_reg_smem) would carry past the size.  Built and read by tests/test_smem_budget_cpu.py.
//   <kernel> <cap> <largest size over the accepted shapes> <shape of the largest> <shapes whose carve passes the size>
#include <cstdio>

#include "forest.cuh"

using namespace b200aa::forest;

alignas(16) static unsigned char smem[kSmemCap];      // the dynamic shared memory's 16-byte alignment

int main()
{
    size_t big = 0;
    int bf = 0, bc = 0, past = 0;
    for (int F = 1; F <= kMaxFeats; ++F)
        for (int C = 1; C <= kMaxClasses; ++C) {
            if (smem_bytes(F, C) > big) {
                big = smem_bytes(F, C);
                bf = F;
                bc = C;
            }
            Tree T{};
            T.F = F;
            T.C = C;
            past += size_t(carve_smem(smem, kThreads, T) - smem) > smem_bytes(F, C);
        }
    printf("forest_build_kernel %zu %zu %d:%d %d\n", kSmemCap, big, bf, bc, past);
    size_t rbig = 0, bbig = 0;
    int rf = 0, bbf = 0, rpast = 0, bpast = 0;
    for (int F = 1; F <= kMaxFeats; ++F) {
        if (reg_smem_bytes(F) > rbig) rbig = reg_smem_bytes(F), rf = F;
        if (boost_smem_bytes(F) > bbig) bbig = boost_smem_bytes(F), bbf = F;
        RegTree T{};
        T.F = F;
        const size_t end = size_t(carve_reg_smem(smem, T) - smem);
        rpast += end > reg_smem_bytes(F);
        bpast += end + size_t(kThreads) * 8 > boost_smem_bytes(F);     // boost_build_kernel's part [kThreads] besides
    }
    printf("forest_reg_build_kernel %zu %zu %d:1 %d\n", kRegSmemCap, rbig, rf, rpast);
    printf("boost_build_kernel %zu %zu %d:1 %d\n", kBoostSmemCap, bbig, bbf, bpast);
    return 0;
}
