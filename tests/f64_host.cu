// Host program for tests/test_f64_cpu.py: runs the float64 path's __host__ __device__ pieces (pyaudioanalysis_b200/csrc/
// f64.cuh) on the CPU in the order the kernels apply them.  Reads commands from stdin, numbers as C hex floats / "inf" /
// "nan"; prints hex floats ("nan" for NaN).
//
//   norm n X (n)                 -> mean, scale of the clip's normalisation record, then the n normalised samples
//   time w Y (w)                 -> zcr, energy, energy entropy of one normalised frame
//   pool F T ratio stepr X (FxT) -> the [2F, M] mid-term matrix
//   fft n RE (n)                 -> re (n), im (n) of the fp64 mixed-radix transform of a real frame
//   spec n Y (n)                 -> |X|[0:K] / K of that transform (f64::magnitude), as the frame kernel writes it
//   specrec n Y (n)              -> the same with twiddles built by recurrence, w^j = w^(j-1) w (a planted defect)
//   tables fs K                  -> the plan's dense [40 x K] mel bank, then the [13 x 40] DCT (b200aa_host::build_mel,
//                                   build_dct: the tables kernel 12's MFCC stage reads)
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/f64.cuh"
#include "../pyaudioanalysis_b200/csrc/rows.cuh"
#include "../pyaudioanalysis_b200/csrc/tables.inl"
#include "host_io.h"

using namespace b200aa;

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "norm")) {
            const int64_t n = rl();
            const std::vector<double> x = rv(size_t(n));
            const double s = f64::np_sum_lanes([&](int64_t i) { return f64::scaled(x[size_t(i)]); }, n);
            const double mean = npy::ddiv(s, double(n));
            double mx = 0.0;
            for (int64_t i = 0; i < n; ++i) {
                const double v = std::fabs(npy::dsub(f64::scaled(x[size_t(i)]), mean));
                mx = (v > mx || v != v) ? v : mx;
            }
            const b200aa_clip_norm_f64 nm{mean, npy::dadd(mx, 1e-10)};
            printf("N");
            pr(nm.mean);
            pr(nm.scale);
            for (int64_t i = 0; i < n; ++i) pr(f64::normalised(x[size_t(i)], nm));
            printf("\n");
        } else if (!strcmp(cmd, "time")) {
            const int w = int(rl());
            const std::vector<double> y = rv(size_t(w));
            int64_t flips = 0;
            for (int i = 1; i < w; ++i) flips += std::abs(f64::sign_of(y[i]) - f64::sign_of(y[i - 1]));
            const double tot = f64::np_sum_lanes([&](int64_t i) { return npy::dmul(y[size_t(i)], y[size_t(i)]); }, w);
            const int blk = w / 10;
            double t[10];
            for (int j = 0; j < 10; ++j) {
                const double e = front::np_sum([&](int64_t i) { const double v = y[size_t(j * blk + i)]; return npy::dmul(v, v); },
                                               blk, true);
                t[j] = f64::entropy_term(e, tot, [](double v) { return std::log2(v); });
            }
            printf("T");
            pr(f64::zcr_of(flips, w));
            pr(f64::energy_of(tot, w));
            pr(f64::entropy_of(t));
            printf("\n");
        } else if (!strcmp(cmd, "pool")) {
            const int F = int(rl());
            const int64_t T = rl(), ratio = rl(), stepr = rl();
            const std::vector<double> X = rv(size_t(F * T));
            const int64_t M = rows::windows_of(T, int(stepr));
            std::vector<double> out(size_t(2 * F * M));
            for (int f = 0; f < F; ++f)
                for (int64_t j = 0; j < M; ++j)
                    f64::mid_window([&](int64_t c) { return X[size_t(f * T + c)]; }, T, j, ratio, stepr,
                                    out[size_t(f * M + j)], out[size_t((F + f) * M + j)]);
            printf("P");
            for (double v : out) pr(v);
            printf("\n");
        } else if (!strcmp(cmd, "tables")) {
            const int fs = int(rl()), K = int(rl());
            std::vector<double> mel, dct;
            b200aa_host::build_mel(fs, K, mel);
            b200aa_host::build_dct(dct);
            printf("M");
            for (double v : mel) pr(v);
            for (double v : dct) pr(v);
            printf("\n");
        } else if (!strcmp(cmd, "fft") || !strcmp(cmd, "spec") || !strcmp(cmd, "specrec")) {
            const int n = int(rl());
            const std::vector<double> re = rv(size_t(n));
            std::vector<f64::Cplx> a(n), b(n), tw(n);
            for (int j = 0; j < n; ++j) {
                a[j] = {re[j], 0.0};
                const double ang = -2.0 * b200aa_host::kPi * double(j) / double(n);
                tw[j] = {std::cos(ang), std::sin(ang)};
                if (!strcmp(cmd, "specrec") && j > 1)
                    tw[j] = {tw[j - 1].x * tw[1].x - tw[j - 1].y * tw[1].y, tw[j - 1].x * tw[1].y + tw[j - 1].y * tw[1].x};
            }
            std::vector<int> radix = b200aa_host::radix_list(n);
            if (n == 1) radix.clear();
            int Ns = 1;
            for (int R : radix) {
                for (int o = 0; o < n; ++o)
                    b[o] = f64::stockham_output([&](int i) { return a[i]; }, o, n, Ns, R, [&](int i) { return tw[i]; });
                std::swap(a, b);
                Ns *= R;
            }
            if (strcmp(cmd, "fft")) {
                printf("S");
                for (int k = 0; k < n / 2; ++k) pr(f64::magnitude(a[k], n / 2));
                printf("\n");
                continue;
            }
            printf("F");
            for (int k = 0; k < n; ++k) pr(a[k].x);
            for (int k = 0; k < n; ++k) pr(a[k].y);
            printf("\n");
        }
    }
    return 0;
}
