// Host program for tests/test_pcm_cpu.py: runs the per-frame conversion of the decode kernel (pyaudioanalysis_b200/csrc/
// pcm.cuh, __host__ __device__) on the CPU.
//
//   pcm_host FORMAT CHANNELS N_FRAMES OUT_DTYPE IN OUT
//
// IN holds N_FRAMES raw frames of a WAV data chunk (B200AA_PCM_* FORMAT, 1 or 2 channels); OUT receives N_FRAMES int16
// (OUT_DTYPE 0) or float32 (1) samples, as the kernel stages them.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/pcm.cuh"

using namespace b200aa;

int main(int argc, char **argv)
{
    if (argc != 7) return 2;
    const int format = atoi(argv[1]), channels = atoi(argv[2]), out_dtype = atoi(argv[4]);
    const long long n = atoll(argv[3]);
    const int block = channels * pcm::sample_bytes(format);
    if (block <= 0) return 2;
    std::vector<unsigned char> in(size_t(n) * block + 16);       // 16-byte aligned frames, as in the arena
    FILE *f = fopen(argv[5], "rb");
    if (!f || fread(in.data(), 1, size_t(n) * block, f) != size_t(n) * block) return 3;
    fclose(f);
    FILE *g = fopen(argv[6], "wb");
    if (!g) return 3;
    for (long long i = 0; i < n; ++i) {
        const unsigned char *frame = in.data() + size_t(i) * block;
        if (out_dtype == 0) {
            const int16_t v = pcm::frame_i16(frame, format);
            fwrite(&v, sizeof v, 1, g);
        } else {
            const float v = pcm::frame_f32(frame, format, channels);
            fwrite(&v, sizeof v, 1, g);
        }
    }
    fclose(g);
    return 0;
}
