// Host harness of the per-(fs, window) tables of the short-term kernels: the status of the mel bank and the chroma operator
// (csrc/tables.inl), the generic kernel's blob (b200aa_host::build_blob), the pair / solo kernels' blob (build_pair_blob) and
// the shared-memory footprint each specialised launch would ask for with those blobs.  Built and read by
// tests/test_rates_cpu.py (nvcc host compile; no GPU needed).
// stdin: lines "fs window n_hops hop..."; stdout per line:
//   T fs window mel_status chroma_status generic_words
//   and, where both tables build (the plan builds the pair blob only then):
//   B words lq ct dct mel_rec mel_w chr          the pair blob's layout
//   W word ...                                   its raw int32 words
//   S kind bytes cap                             pair (pair windows) / solo_features, solo_chroma (solo windows)
//   F hop runs bytes                             CTA windows, per hop: bytes with run staging (runs 1, when the launcher
//                                                can pick it) and without (runs 0); the launcher's cap is 110 KB
#include <cstdio>
#include <sstream>
#include <string>
#include <iostream>
#define B200AA_LAYOUT_ONLY 1      // skip the launchers: they would instantiate every kernel
#include "../pyaudioanalysis_b200/csrc/fast_kernel.cuh"
#include "../pyaudioanalysis_b200/csrc/solo_kernel.cuh"
#include "../pyaudioanalysis_b200/csrc/tables.inl"
using namespace b200aa;

static size_t pair_bytes(int R, int words)
{
    switch (R) {
    case 10: return pair_smem_bytes<10>(words);
    case 15: return pair_smem_bytes<15>(words);
    case 16: return pair_smem_bytes<16>(words);
    case 20: return pair_smem_bytes<20>(words);
    case 25: return pair_smem_bytes<25>(words);
    case 30: return pair_smem_bytes<30>(words);
    case 32: return pair_smem_bytes<32>(words);
    default: return 0;
    }
}

template <int L, int R2>
static void solo_row(int words)
{
    printf("S solo_features %zu %d\n", solo_smem_bytes<L, R2, kModeFeatures>(words), kSoloCtaCap);
    printf("S solo_chroma %zu %d\n", solo_smem_bytes<L, R2, kModeChromagram>(words), 113 * 1024);
}

template <int R1, int R2>
static void fast_row(int hop, int words)
{
    constexpr int N = 2 * R1 * R2;
    if (N % 80 == 0 && hop % 8 == 0) printf("F %d 1 %zu\n", hop, fast_smem_bytes<R1, R2, B200AA_FAST_G>(hop, words, true));
    printf("F %d 0 %zu\n", hop, fast_smem_bytes<R1, R2, B200AA_FAST_G>(hop, words, false));
}

static void fast_rows(int window, int hop, int words)
{
    switch (window) {
    case 800: fast_row<20, 20>(hop, words); break;
    case 882: fast_row<21, 21>(hop, words); break;
    case 400: fast_row<20, 10>(hop, words); break;
    case 480: fast_row<20, 12>(hop, words); break;
    case 600: fast_row<20, 15>(hop, words); break;
    case 320: fast_row<16, 10>(hop, words); break;
    case 640: fast_row<20, 16>(hop, words); break;
    default: break;
    }
}

int main()
{
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        int fs = 0, w = 0, nh = 0;
        if (!(in >> fs >> w >> nh)) continue;
        std::vector<int> hops(nh);
        for (int &h : hops) in >> h;
        const int K = w / 2;
        std::vector<double> mel, chr, dct;
        const int rc_mel = b200aa_host::build_mel(fs, K, mel);
        const int rc_chr = b200aa_host::build_chroma(fs, K, chr);
        b200aa_host::build_dct(dct);
        std::vector<int> gblob;
        BlobLayout gbl{};
        b200aa_host::build_blob(fs, K, gblob, gbl);
        printf("T %d %d %d %d %d\n", fs, w, rc_mel, rc_chr, gbl.words);
        int r1 = 0, r2 = 0;
        if (fast_shape_for_window(w, &r1, &r2))
            for (int h : hops) fast_rows(w, h, gbl.words);
        if (rc_mel != B200AA_OK || rc_chr != B200AA_OK) continue;
        std::vector<int> pblob;
        PairBlobLayout pbl{};
        build_pair_blob(mel, chr, dct, K, pblob, pbl);
        printf("B %d %d %d %d %d %d %d\n", pbl.words, pbl.lq, pbl.ct, pbl.dct, pbl.mel_rec, pbl.mel_w, pbl.chr);
        printf("W");
        for (int v : pblob) printf(" %d", v);
        printf("\n");
        if (const int R = pair_r_for_window(w)) printf("S pair %zu %d\n", pair_bytes(R, pbl.words), kPairCtaCap);
        switch (w) {
        case 882: solo_row<21, 21>(pbl.words); break;
        case 400: solo_row<20, 10>(pbl.words); break;
        case 600: solo_row<20, 15>(pbl.words); break;
        default: break;
        }
    }
    return 0;
}
