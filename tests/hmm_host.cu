// Host program for tests/test_hmm_cpu.py: runs the __host__ __device__ pieces of kernel 7 (pyaudioanalysis_b200/csrc/hmm.cuh)
// on the CPU in the order the kernels apply them.  Reads commands from stdin, numbers as C hex floats / "inf" / "nan";
// prints hex floats ("nan" for NaN).
//
//   stats n pairwise x (n)                                  -> sum mean ssq std
//   emission F n pairwise konst mu (F) var (F) x (n x F)    -> the n emissions
//   viterbi C n log_start (C) log_trans (C x C) e (n x C)   -> the n states
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/hmm.cuh"
#include "host_io.h"

using namespace b200aa;

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "stats")) {
            const int64_t n = rl();
            const bool pw = rl() != 0;
            const std::vector<double> x = rv(size_t(n));
            const hmm::ClassStats s = hmm::class_stats([&](int64_t i) { return x[size_t(i)]; }, n, pw);
            printf("stats");
            pr(s.sum);
            pr(s.mean);
            pr(s.ssq);
            pr(s.std);
            printf("\n");
        } else if (!strcmp(cmd, "emission")) {
            const int F = int(rl());
            const int64_t n = rl();
            const bool pw = rl() != 0;
            const double konst = rd();
            const std::vector<double> mu = rv(size_t(F)), var = rv(size_t(F)), x = rv(size_t(n) * F);
            printf("emission");
            for (int64_t t = 0; t < n; ++t)
                pr(hmm::emission([&](int64_t f) { return x[size_t(t) * F + f]; }, mu.data(), var.data(), F, konst, pw));
            printf("\n");
        } else if (!strcmp(cmd, "viterbi")) {
            const int C = int(rl());
            const int64_t n = rl();
            const std::vector<double> ls = rv(size_t(C)), la = rv(size_t(C) * C), e = rv(size_t(n) * C);
            std::vector<double> prev(C), cur(C);
            std::vector<int32_t> bp(size_t(n) * C, 0);
            for (int j = 0; j < C; ++j) cur[j] = hmm::dadd(ls[j], e[j]);
            for (int64_t t = 1; t < n; ++t) {
                prev.swap(cur);
                for (int j = 0; j < C; ++j)
                    cur[j] = hmm::step([&](int32_t i) { return prev[i]; }, [&](int32_t i) { return la[size_t(i) * C + j]; }, C,
                                       e[size_t(t) * C + j], bp[size_t(t) * C + j]);
            }
            std::vector<int32_t> path(n);
            path[n - 1] = hmm::last_state([&](int32_t i) { return cur[i]; }, C);
            for (int64_t t = n - 1; t > 0; --t) path[t - 1] = bp[size_t(t) * C + path[t]];
            printf("viterbi");
            for (int64_t t = 0; t < n; ++t) printf(" %d", path[t]);
            printf("\n");
        } else {
            return 2;
        }
    }
    return 0;
}
