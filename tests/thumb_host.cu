// Host program for tests/test_thumbnail_cpu.py: runs kernel 10's __host__ __device__ pieces
// (pyaudioanalysis_b200/csrc/thumb.cuh) on the CPU in the order the kernels apply them.  Reads commands from stdin, numbers
// as C hex floats / "inf" / "nan"; prints hex floats ("nan" for NaN).
//
//   sim T F X (T x F)                    -> S (T x T): row norms, the two-accumulator dot, similarity, 1.0 on the diagonal
//   thumb T F m gap lo hi X (T x F)      -> i1 i2 j1 j2, then the masked C (R x R): S, the NaN windows and box rule, the
//                                           diagonal sums, the min key, the masks, the argmax key and the walk
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/thumb.cuh"
#include "host_io.h"

using namespace b200aa;

static std::vector<double> similarity_matrix(const std::vector<double> &X, int64_t T, int F)
{
    std::vector<double> nrm(T), S(size_t(T * T));
    for (int64_t r = 0; r < T; ++r) {
        const double *x = &X[size_t(r * F)];
        nrm[r] = npy::dsqrt(thumb::dot([x](int k) { return npy::dmul(x[k], x[k]); }, F));
    }
    for (int64_t u = 0; u < T; ++u) {
        S[size_t(u * T + u)] = 1.0;
        for (int64_t v = u + 1; v < T; ++v) {
            const double *x = &X[size_t(u * F)], *y = &X[size_t(v * F)];
            const double d = thumb::dot([x, y](int k) { return npy::dmul(x[k], y[k]); }, F);
            S[size_t(u * T + v)] = S[size_t(v * T + u)] = thumb::similarity(d, nrm[u], nrm[v]);
        }
    }
    return S;
}

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "sim")) {
            const int64_t T = rl();
            const int F = int(rl());
            const std::vector<double> S = similarity_matrix(rv(size_t(T * F)), T, F);
            printf("S");
            for (double s : S) pr(s);
            printf("\n");
        } else if (!strcmp(cmd, "thumb")) {
            const int64_t T = rl();
            const int F = int(rl()), m = int(rl());
            const double gap = rd();
            const int64_t lo = rl(), hi = rl();
            const std::vector<double> S = similarity_matrix(rv(size_t(T * F)), T, F);
            const int64_t R = T - m + 1;
            bool any_nan = false;
            for (double s : S) any_nan |= s != s;
            std::vector<unsigned char> Hn(size_t(T * R), 0);       // thumb_nan_window_kernel
            if (any_nan)
                for (int64_t a = 0; a < T; ++a)
                    for (int64_t j = 0; j < R; ++j)
                        for (int k = 0; k < m; ++k) Hn[size_t(a * R + j)] |= S[size_t(a * T + j + k)] != S[size_t(a * T + j + k)];
            std::vector<double> C(size_t(R * R));
            uint64_t kmin = ~uint64_t(0);
            auto at = [&](int64_t a, int64_t b) { return S[size_t(a * T + b)]; };
            for (int64_t i = 0; i < R; ++i)                         // thumb_filter_kernel
                for (int64_t j = i; j < R; ++j) {
                    double c = thumb::diag_sum(at, i, j, m);
                    bool nan = false;
                    for (int k = 0; k < m; ++k) nan |= Hn[size_t((i + k) * R + j)] != 0;
                    if (nan) c = thumb::double_of(0x7ff8000000000000ull);
                    C[size_t(i * R + j)] = C[size_t(j * R + i)] = c;
                    kmin = std::min(kmin, thumb::min_key(c));
                }
            const double min_sm = thumb::min_value(kmin);
            uint64_t bk = 0;
            int64_t bi = INT64_MAX;
            for (int64_t e = 0; e < R * R; ++e) {                   // thumb_mask_kernel, in reverse: the key decides
                const int64_t e2 = R * R - 1 - e, i = e2 / R, j = e2 % R;
                if (thumb::masked(i, j, gap, lo, hi)) C[size_t(e2)] = min_sm;
                const uint64_t k = thumb::max_key(C[size_t(e2)]);
                if (thumb::better(k, e2, bk, bi)) {
                    bk = k;
                    bi = e2;
                }
            }
            int64_t idx[4];
            thumb::walk([&](int64_t i, int64_t j) { return C[size_t(i * R + j)]; }, R, bi / R, bi % R, m, idx);
            printf("I %lld %lld %lld %lld\nC", (long long)idx[0], (long long)idx[1], (long long)idx[2], (long long)idx[3]);
            for (double c : C) pr(c);
            printf("\n");
        } else {
            fprintf(stderr, "unknown command %s\n", cmd);
            return 1;
        }
    }
    return 0;
}
