// Host program for tests/test_knn_cv_cpu.py: runs the __host__ __device__ pieces of kernel 6's first step
// (pyaudioanalysis_b200/csrc/knn_cv.cuh) on the CPU, column by column as the gather kernel applies them.  Reads commands
// from stdin, numbers as C hex floats; prints results as hex floats ("nan" for NaN).
//
//   fit n m F  train (n x F)  test (m x F)   -> "mean" F values, "scale" F values, "train" n x F and "test" m x F
//                                               standardised values (row-major)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/knn_cv.cuh"
#include "host_io.h"

using namespace b200aa;

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (strcmp(cmd, "fit")) return 2;
        const int64_t n = rl(), m = rl();
        const int F = int(rl());
        const std::vector<double> tr = rv(size_t(n) * F), te = rv(size_t(m) * F);
        std::vector<knn::Scale> s(F);
        for (int j = 0; j < F; ++j) s[j] = knn::scaler_fit([&](int64_t i) { return tr[size_t(i) * F + j]; }, n);
        printf("mean");
        for (int j = 0; j < F; ++j) pr(s[j].mean);
        printf("\nscale");
        for (int j = 0; j < F; ++j) pr(s[j].scale);
        printf("\ntrain");
        for (size_t e = 0; e < tr.size(); ++e) pr(knn::standardise(tr[e], s[e % F]));
        printf("\ntest");
        for (size_t e = 0; e < te.size(); ++e) pr(knn::standardise(te[e], s[e % F]));
        printf("\n");
    }
    return 0;
}
