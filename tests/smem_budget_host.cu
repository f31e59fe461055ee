// Host-side print of the shared-memory footprint of the CTA kernel per (window, hop) shape and of the pair kernel per window
// (csrc/fast_kernel.cuh: fast_smem_bytes), and of the generic kernel's frames per group for the (fs, window) pairs given on
// the command line (csrc/generic_kernel.cuh: generic_group) at the size of the tables blob their plan builds.  Built and read by
// tests/test_smem_budget_cpu.py; no GPU needed.
#include <cstdio>
#include <cstdlib>
#define B200AA_LAYOUT_ONLY 1      // skip the launchers: they would instantiate every kernel
#include "../pyaudioanalysis_b200/csrc/fast_kernel.cuh"
#include "../pyaudioanalysis_b200/csrc/pair_kernel.cuh"
#include "../pyaudioanalysis_b200/csrc/generic_kernel.cuh"
#include "../pyaudioanalysis_b200/csrc/tables.inl"
using namespace b200aa;

template <int R1, int R2>
static void row(int step, int blob_words)
{
    constexpr int N = 2 * R1 * R2;
    const bool runs = (N % 80 == 0) && (step % 8 == 0);
    printf("fast %d %d %d %zu\n", N, step, int(runs), fast_smem_bytes<R1, R2, B200AA_FAST_G>(step, blob_words, runs));
}

int main(int argc, char **argv)
{
    // generic kernel, per "fs:window" argument: transform points, the blob the plan builds (b200aa_host::build_blob), and
    // the frames per group with that blob, with 256 words less and with 256 words more, then the shared-memory bytes
    for (int i = 1; i < argc; ++i) {
        int fs = 0, w = 0;
        if (sscanf(argv[i], "%d:%d", &fs, &w) != 2) return 1;
        const int K = w / 2, Kp = (K + 3) & ~3, Nc = (w % 2 == 0) ? w / 2 : w;
        std::vector<int> blob;
        BlobLayout bl{};
        b200aa_host::build_blob(fs, K, blob, bl);
        const int words = bl.words, g = generic_group(Nc, Kp, words);
        printf("generic %d %d %d %d %d %d %d %zu\n", fs, w, Nc, words, generic_group(Nc, Kp, words > 256 ? words - 256 : 0), g,
               generic_group(Nc, Kp, words + 256), generic_smem_bytes(g ? g : 1, Nc, Kp, words, g != 0));
    }
    // mel + DCT + chroma blob: the largest over the supported (fs, window) pairs (6 854 Hz, window 1024: the lowest rate whose
    // mel bank builds has the longest filters; tests/test_rates_cpu.py: GENERIC_WORDS_MAX)
    const int words = 1832;
    row<20, 20>(400, words); row<20, 20>(800, words); row<20, 20>(160, words);
    row<21, 21>(441, words); row<21, 21>(882, words);
    row<20, 10>(160, words); row<20, 10>(200, words); row<20, 10>(400, words);
    row<20, 12>(240, words); row<20, 12>(160, words);
    row<20, 15>(300, words);
    row<16, 10>(160, words); row<16, 10>(320, words);
    row<20, 16>(320, words); row<20, 16>(160, words);
    // pair kernel: bytes per CTA with the largest pair blob (2 232 words = 8.7 KB at 6 854 Hz, window 1024;
    // tests/test_rates_cpu.py: PAIR_WORDS_MAX) and warps per CTA
    const int pwords = 2232;
    printf("pair %d %d %zu\n", 320, pair_warps<10>(), pair_smem_bytes<10>(pwords));
    printf("pair %d %d %zu\n", 480, pair_warps<15>(), pair_smem_bytes<15>(pwords));
    printf("pair %d %d %zu\n", 512, pair_warps<16>(), pair_smem_bytes<16>(pwords));
    printf("pair %d %d %zu\n", 640, pair_warps<20>(), pair_smem_bytes<20>(pwords));
    printf("pair %d %d %zu\n", 800, pair_warps<25>(), pair_smem_bytes<25>(pwords));
    printf("pair %d %d %zu\n", 960, pair_warps<30>(), pair_smem_bytes<30>(pwords));
    printf("pair %d %d %zu\n", 1024, pair_warps<32>(), pair_smem_bytes<32>(pwords));
    return 0;
}
