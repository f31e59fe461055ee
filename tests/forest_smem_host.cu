// Host-side print of kernel 13's dynamic shared-memory sizes (pyaudioanalysis_b200/csrc/forest.cuh: smem_bytes,
// reg_smem_bytes, boost_smem_bytes) at every shape the launchers accept, F in 1 .. kMaxFeats and C in 1 .. kMaxClasses,
// against the caps the launchers set as the kernels' limits.  Built and read by tests/test_smem_budget_cpu.py.
//   <kernel> <cap> <largest size over the accepted shapes> <shape of the largest>
#include <cstdio>

#include "forest.cuh"

using namespace b200aa::forest;

int main()
{
    size_t big = 0;
    int bf = 0, bc = 0;
    for (int F = 1; F <= kMaxFeats; ++F)
        for (int C = 1; C <= kMaxClasses; ++C)
            if (smem_bytes(F, C) > big) {
                big = smem_bytes(F, C);
                bf = F;
                bc = C;
            }
    printf("forest_build_kernel %zu %zu %d:%d\n", kSmemCap, big, bf, bc);
    size_t rbig = 0, bbig = 0;
    int rf = 0, bbf = 0;
    for (int F = 1; F <= kMaxFeats; ++F) {
        if (reg_smem_bytes(F) > rbig) rbig = reg_smem_bytes(F), rf = F;
        if (boost_smem_bytes(F) > bbig) bbig = boost_smem_bytes(F), bbf = F;
    }
    printf("forest_reg_build_kernel %zu %zu %d:1\n", kRegSmemCap, rbig, rf);
    printf("boost_build_kernel %zu %zu %d:1\n", kBoostSmemCap, bbig, bbf);
    return 0;
}
