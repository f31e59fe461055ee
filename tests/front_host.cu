// Host program for tests/test_front_cpu.py: runs kernel 11's __host__ __device__ pieces (pyaudioanalysis_b200/csrc/front.cuh)
// on the CPU in the order the kernels apply them.  Reads commands from stdin, numbers as C hex floats / "inf" / "nan";
// prints hex floats ("nan" for NaN).
//
//   scale n D pairwise X (n x D)   -> mean (D), scale (D), the +-inf flag, then (X - mean) / scale (n x D)
//   outlier M D X (M x D)          -> dist_all (D), mean, then the kept flags (D): kernel 9's chain between the columns
//   pool F T r X (F x T)           -> the pooled [2F, T] matrix
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/front.cuh"
#include "host_io.h"

using namespace b200aa;

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "scale")) {
            const int64_t n = rl();
            const int D = int(rl());
            const bool pairwise = rl() != 0;
            const std::vector<double> X = rv(size_t(n * D));
            std::vector<knn::Scale> s(D);
            bool any_inf = false;
            for (int j = 0; j < D; ++j) {
                bool inf;
                s[j] = front::scaler_fit([&](int64_t i) { return X[size_t(i * D + j)]; }, n, pairwise, inf);
                any_inf |= inf;
            }
            printf("S");
            for (int j = 0; j < D; ++j) pr(s[j].mean);
            for (int j = 0; j < D; ++j) pr(s[j].scale);
            pr(any_inf ? 1.0 : 0.0);
            for (int64_t i = 0; i < n; ++i)
                for (int j = 0; j < D; ++j) pr(knn::standardise(X[size_t(i * D + j)], s[j]));
            printf("\n");
        } else if (!strcmp(cmd, "outlier")) {
            const int64_t M = rl();
            const int D = int(rl());
            const std::vector<double> X = rv(size_t(M * D));
            std::vector<double> dist(size_t(D) * D), dist_all(D);
            for (int u = 0; u < D; ++u)
                for (int v = 0; v < D; ++v) {
                    double a = 0.0;                     // cluster_dist_kernel's chain, from 0.0
                    for (int64_t f = 0; f < M; ++f) a = knn::dist_step(a, X[size_t(f * D + u)], X[size_t(f * D + v)]);
                    dist[size_t(u) * D + v] = npy::dsqrt(a);
                }
            for (int j = 0; j < D; ++j)
                dist_all[j] = front::column_sum([&](int i, int c) { return dist[size_t(i) * D + c]; }, D, j);
            const double mean = front::outlier_mean([&](int64_t j) { return dist_all[size_t(j)]; }, D);
            const double thr = front::outlier_threshold(mean);
            printf("O");
            for (double d : dist_all) pr(d);
            pr(mean);
            for (double d : dist_all) pr(d < thr ? 1.0 : 0.0);
            printf("\n");
        } else if (!strcmp(cmd, "pool")) {
            const int F = int(rl());
            const int64_t T = rl(), r = rl();
            const std::vector<double> X = rv(size_t(F * T));
            std::vector<double> out(size_t(2 * F * T));
            for (int f = 0; f < F; ++f)
                for (int64_t i = 0; i < T; ++i) {
                    const double *w = &X[size_t(f * T + i)];
                    front::pool_window([w](int64_t k) { return w[k]; }, r < T - i ? r : T - i, out[size_t(f * T + i)],
                                       out[size_t((F + f) * T + i)]);
                }
            printf("P");
            for (double v : out) pr(v);
            printf("\n");
        }
    }
    return 0;
}
