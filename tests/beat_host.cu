// Host program for tests/test_beat_cpu.py: runs the __host__ __device__ pieces of kernel 4 (pyaudioanalysis_b200/csrc/beat.cuh)
// on the CPU.  Reads commands from stdin, numbers as C hex floats / "inf" / "nan"; prints results as hex floats.
//
//   sum N v_0 .. v_{N-1} K n_1 .. n_K   -> per n: the pairwise sum of v[:n] serially, split over 32 lanes and over 256 lanes
//   peaks C T delta v_0 .. v_{T-1}      -> peak positions of the chunked scan with chunk length C
//   beat C F T window v (F x T, rows)   -> bpm ratio of the whole per-clip computation with chunk length C
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/beat.cuh"

using namespace b200aa;

static double rd()
{
    char buf[64];
    if (scanf("%63s", buf) != 1) exit(2);
    return strtod(buf, nullptr);
}
static long long rl() { return (long long)rd(); }
static void pr(double x)
{
    if (x != x) printf(" nan");
    else printf(" %a", x);
}

template <class G>
static double lanes_sum(const G &get, int64_t n, int64_t nz, int levels)
{
    std::vector<double> s(size_t(1) << levels);
    for (size_t k = 0; k < s.size(); ++k) {
        int64_t off, len;
        beat::pairwise_part(n, levels, int(k), off, len);
        s[k] = beat::pairwise_sum(get, off, len, nz);
    }
    for (size_t o = 1; o < s.size(); o <<= 1)
        for (size_t k = 0; k < s.size(); k += 2 * o) s[k] = beat::dadd(s[k], s[k + o]);
    return s[0];
}

// the three phases of the kernel's scan, run chunk by chunk; emit(p) for every peak, in order
template <class V, class E>
static void chunked_scan(const V &v, int32_t T, int32_t C, double delta, const E &emit)
{
    const int32_t nch = (T + C - 1) / C;
    std::vector<beat::Chunk> rec(nch);
    for (int32_t c = 0; c < nch; ++c) rec[c] = beat::spec_chunk(v, c * C, std::min(T, (c + 1) * C), delta);
    if (nch > 0) {
        beat::State s = rec[0].s;
        int32_t last = rec[0].last;
        for (int32_t c = 1; c < nch; ++c) {
            const beat::Chunk spec = rec[c];
            rec[c].s = s;
            rec[c].last = last;
            beat::fixup_chunk(v, c * C, std::min(T, (c + 1) * C), delta, spec, s, last);
        }
    }
    for (int32_t c = 0; c < nch; ++c)
        beat::scan_chunk(v, c * C, std::min(T, (c + 1) * C), delta, c ? rec[c].s : beat::fresh(), emit);
}

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "sum")) {
            const int64_t N = rl();
            std::vector<double> v(N);
            for (auto &x : v) x = rd();
            auto get = [&](int64_t i) { return v[i]; };
            const int64_t K = rl();
            for (int64_t j = 0; j < K; ++j) {
                const int64_t n = rl();
                printf("sum %lld", (long long)n);
                pr(beat::pairwise_sum(get, 0, n, n));
                pr(lanes_sum(get, n, n, 5));
                pr(lanes_sum(get, n, n, 8));
                printf("\n");
            }
        } else if (!strcmp(cmd, "peaks")) {
            const int32_t C = int32_t(rl()), T = int32_t(rl());
            const double delta = rd();
            std::vector<double> v(T);
            for (auto &x : v) x = rd();
            printf("peaks");
            chunked_scan([&](int32_t i) { return v[i]; }, T, C, delta, [](int32_t p) { printf(" %d", p); });
            printf("\n");
        } else if (!strcmp(cmd, "beat")) {
            const int32_t C = int32_t(rl()), F = int32_t(rl()), T = int32_t(rl());
            const double w = rd();
            std::vector<double> st(size_t(F) * T);
            for (auto &x : st) x = rd();
            const int64_t mbt = int64_t(std::nearbyint(2.0 / w));
            const int64_t nb = std::min<int64_t>(mbt, std::max(T - 1, 0));
            std::vector<unsigned> cnt(size_t(beat::kRows) * nb, 0u);
            for (int r = 0; r < beat::kRows; ++r) {
                const double *row = st.data() + size_t(beat::row_index(r)) * T;
                const int64_t n = T > 1 ? T - 1 : 0;
                const double delta = beat::threshold(
                    lanes_sum([&](int64_t i) { return std::fabs(beat::dsub(row[i], row[i + 1])); }, n, n, 5), T);
                int32_t last = -1;
                chunked_scan([&](int32_t i) { return row[i]; }, T, C, delta, [&](int32_t p) {
                    if (last >= 0 && p - last >= 1 && p - last <= mbt) cnt[size_t(r) * nb + (p - last - 1)]++;
                    last = p;
                });
            }
            auto hist = [&](int64_t k) {
                double h = 0.0;
                for (int r = 0; r < beat::kRows; ++r) h = beat::dadd(h, beat::ddiv(double(cnt[size_t(r) * nb + k]), double(T)));
                return h;
            };
            double bv = 0.0;
            int64_t bk = 0;
            for (int64_t k = 0; k < nb; ++k)
                if (hist(k) > bv) { bv = hist(k); bk = k; }
            const double s = lanes_sum(hist, mbt, nb, 5);
            printf("beat");
            pr(beat::ddiv(60.0, beat::dmul(double(bk + 1), w)));
            pr(T == 0 ? NAN : beat::ddiv(bv, beat::dadd(s, 0.00000001)));
            printf("\n");
        } else {
            return 2;
        }
    }
    return 0;
}
