// libb200aa.so -- PCM WAV decode.
#include <algorithm>

#include "../../include/b200aa.h"
#include "entry.h"
#include "pcm.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// PCM WAV decode (csrc/pcm.cuh): raw data chunks of a byte arena -> the [B, N] int16 / float32 ragged batch
// ------------------------------------------------------------------------------------------------
extern "C" int b200aa_decode_pcm(const void *d_arena, int64_t arena_bytes, const b200aa_pcm_clip *h_clips, int64_t n_clips,
                                 int out_dtype, void *d_out, int64_t n_out, int64_t out_stride, void *stream)
{
    NvtxRange nvtx_("b200aa_decode_pcm");
    REFUSE_CAPTURE(stream, "b200aa_decode_pcm", kWhyHostArrays);
    if (!d_arena || !h_clips || !d_out || arena_bytes < 0 || n_clips < 0 || n_out < 0 || out_stride < n_out ||
        (out_dtype != B200AA_DTYPE_I16 && out_dtype != B200AA_DTYPE_F32))
        return B200AA_ERR_INVALID;
    for (int64_t b = 0; b < n_clips; ++b) {
        const b200aa_pcm_clip &c = h_clips[b];
        const int64_t bytes = pcm::sample_bytes(c.format);
        if (bytes == 0 || (c.channels != 1 && c.channels != 2) || c.offset < 0 || c.offset % 16 || c.n_frames < 0 ||
            c.n_frames > n_out)
            return B200AA_ERR_INVALID;
        if (out_dtype == B200AA_DTYPE_I16 && (c.channels != 1 || (c.format != B200AA_PCM_U8 && c.format != B200AA_PCM_S16)))
            return B200AA_ERR_INVALID;
        const int64_t block = c.channels * bytes;
        if (c.offset > arena_bytes || c.n_frames > (arena_bytes - c.offset) / block ||
            (c.n_frames * block + 15) / 16 * 16 > arena_bytes - c.offset)      // the kernel reads whole 16-byte words
            return B200AA_ERR_INVALID;
    }
    if (n_clips == 0 || n_out == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t clip_bytes = size_t(n_clips) * sizeof(b200aa_pcm_clip);
    const int64_t tiles = (n_out + pcm::kTile - 1) / pcm::kTile;
    const int64_t items = n_clips * tiles;
    const unsigned grid = unsigned(std::min<int64_t>(items, int64_t(1) << 30));
    StreamScratch scratch(st);
    int rc = scratch.alloc(clip_bytes);
    if (rc != B200AA_OK) return rc;
    const b200aa_pcm_clip *d_clips = static_cast<const b200aa_pcm_clip *>(scratch.get());
    const cudaError_t e = cudaMemcpyAsync(scratch.get(), h_clips, clip_bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpyAsync");
    const unsigned char *arena = static_cast<const unsigned char *>(d_arena);
    auto decode = [&](auto *out) {
        pcm::decode_kernel<<<grid, pcm::kThreads, 0, st>>>(arena, d_clips, items, tiles, n_out, out_stride, out);
    };
    if (out_dtype == B200AA_DTYPE_I16) decode(static_cast<int16_t *>(d_out));
    else decode(static_cast<float *>(d_out));
    return scratch.done(launched("pcm::decode_kernel"));
}
