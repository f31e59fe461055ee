// Host harness of csrc/rows.cuh: the row arithmetic of spectrogram() / chromagram() that the entry points, the ragged row
// kernels and b200aa_row_counts share.  Built and run by tests/test_rows_cpu.py (nvcc host compile; no GPU needed).
// stdin: lines "w s n_max"; stdout per line: "max_clipped", then one line per n = 0 .. n_max:
//   n  spec_R spec_n_it spec_n_full spec_refused  chroma_R chroma_n_it chroma_n_full chroma_refused
#include <cstdio>

#include "../pyaudioanalysis_b200/csrc/rows.cuh"

int main()
{
    int w, s;
    long long n_max;
    while (scanf("%d %d %lld", &w, &s, &n_max) == 3) {
        printf("%lld\n", (long long)b200aa::rows::max_clipped(w, s));
        for (long long n = 0; n <= n_max; ++n) {
            const b200aa::rows::Rows a = b200aa::rows::spectrogram(n, w, s), c = b200aa::rows::chromagram(n, w, s);
            printf("%lld %lld %lld %lld %d %lld %lld %lld %d\n", n, (long long)a.R, (long long)a.n_it, (long long)a.n_full,
                   int(a.refused), (long long)c.R, (long long)c.n_it, (long long)c.n_full, int(c.refused));
        }
    }
    return 0;
}
