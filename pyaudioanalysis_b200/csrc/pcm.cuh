// PCM WAV decode on the device: the raw data chunks of a batch of WAV files, read straight from disk into one byte arena,
// become the [B, N] int16 / float32 ragged batch the feature path takes.  Every frame converts to exactly what
// `_as_clip(stereo_to_mono(scipy.io.wavfile.read(path)[1]))` stages on the host (audioBasicIO.py:86-110, :156-168):
//
//   format  scipy dtype           mono                     stereo (L = channel 0, R = channel 1)
//   U8      uint8                 int16 u                  f32(R/2 + L/2) in double: exact
//   S16     int16                 int16 x                  f32(R/2 + L/2) in double: exact
//   S24     int32 (bytes << 8)    f32, exact               f32(R/2 + L/2) in double: the sum is exact, one rounding
//   S32     int32                 f32 RN                   f32(R/2 + L/2) in double: the sum is exact, one rounding
//   F32     float32               bits unchanged           RN(RN(R * 0.5f) + RN(L * 0.5f)): NumPy keeps float32 for arr / 2
//   F64     float64               f32 RN                   f32(RN(R * 0.5 + L * 0.5))
//
// x / 2 and x * 0.5 are the same correctly rounded value, subnormals included.  Every operation is an explicit _rn
// intrinsic on the device, so nothing contracts into an FMA; the library is built without fast math, so float32
// subnormals are kept.  __host__ __device__: tests/pcm_host.cu runs the same conversion on the CPU.
#pragma once
#include <cstdint>
#include <cstring>

namespace b200aa {
namespace pcm {

// bytes per sample of each B200AA_PCM_* format, in the header's order (U8, S16, S24, S32, F32, F64)
__host__ __device__ inline int sample_bytes(int format)
{
    switch (format) {
    case 0: return 1;
    case 1: return 2;
    case 2: return 3;
    case 3: return 4;
    case 4: return 4;
    case 5: return 8;
    default: return 0;
    }
}

// little-endian load of a naturally aligned sample (a slot starts 16-byte aligned and frames are `block` bytes apart)
template <typename T>
__host__ __device__ inline T load(const unsigned char *p)
{
#ifdef __CUDA_ARCH__
    return *reinterpret_cast<const T *>(p);
#else
    T v;
    std::memcpy(&v, p, sizeof(T));
    return v;
#endif
}

// integer sample of channel c as scipy returns it (S24: the three bytes left-justified in an int32)
__host__ __device__ inline int32_t int_sample(const unsigned char *frame, int format, int c)
{
    switch (format) {
    case 0: return int32_t(frame[c]);
    case 1: return int32_t(load<int16_t>(frame + 2 * c));
    case 2: {
        const unsigned char *s = frame + 3 * c;
        return int32_t((uint32_t(s[0]) << 8) | (uint32_t(s[1]) << 16) | (uint32_t(s[2]) << 24));
    }
    default: return load<int32_t>(frame + 4 * c);
    }
}

__host__ __device__ inline double dadd(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline double dmul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float fadd(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline float fmul(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float d2f(double x)
{
#ifdef __CUDA_ARCH__
    return __double2float_rn(x);
#else
    return float(x);
#endif
}
__host__ __device__ inline float i2f(int32_t x)
{
#ifdef __CUDA_ARCH__
    return __int2float_rn(x);
#else
    return float(x);
#endif
}

// one frame of a file staged as float32 (every flavour but mono U8 / S16)
__host__ __device__ inline float frame_f32(const unsigned char *frame, int format, int channels)
{
    if (format == 4) {
        const float l = load<float>(frame);
        if (channels == 1) return l;
        return fadd(fmul(load<float>(frame + 4), 0.5f), fmul(l, 0.5f));
    }
    if (format == 5) {
        const double l = load<double>(frame);
        if (channels == 1) return d2f(l);
        return d2f(dadd(dmul(load<double>(frame + 8), 0.5), dmul(l, 0.5)));
    }
    const int32_t l = int_sample(frame, format, 0);
    if (channels == 1) return i2f(l);
    return d2f(dadd(dmul(double(int_sample(frame, format, 1)), 0.5), dmul(double(l), 0.5)));
}

// one frame of a mono U8 / S16 file, staged as int16
__host__ __device__ inline int16_t frame_i16(const unsigned char *frame, int format)
{
    return int16_t(int_sample(frame, format, 0));
}

constexpr int kTile = 1024;       // frames per work item
constexpr int kThreads = 256;

#ifdef __CUDACC__
// One work item = (clip b, tile t) = output elements [t * kTile, (t + 1) * kTile) of row b; items run grid-stride in one
// launch, so the clip count is not bound by a grid dimension.  The tile's bytes (at most kTile * 16: stereo float64) come
// in as coalesced 16-byte words of the clip's slot into shared memory; every thread then converts frames i, i + 256, ...
// and stores them coalesced.  Elements past the clip's frames are zero.
template <typename OUT, typename Clip>
__global__ void __launch_bounds__(kThreads) decode_kernel(const unsigned char *__restrict__ arena, const Clip *__restrict__ clips,
                                                          int64_t n_items, int64_t tiles_per_row, int64_t n_out,
                                                          int64_t out_stride, OUT *__restrict__ out)
{
    __shared__ uint4 buf[kTile];
    const unsigned char *bytes = reinterpret_cast<const unsigned char *>(buf);
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int64_t b = item / tiles_per_row;
        const int64_t f0 = (item - b * tiles_per_row) * kTile;
        const Clip c = clips[b];
        const int block = c.channels * sample_bytes(c.format);
        const int64_t left = c.n_frames - f0;
        const int nf = left <= 0 ? 0 : (left < kTile ? int(left) : kTile);
        const int64_t words = (int64_t(nf) * block + 15) / 16;     // inside the zero-padded slot: f0 * block is 16-aligned
        const uint4 *src = reinterpret_cast<const uint4 *>(arena + c.offset + f0 * block);
        for (int64_t w = threadIdx.x; w < words; w += kThreads) buf[w] = src[w];
        __syncthreads();
        OUT *row = out + b * out_stride;
        for (int i = threadIdx.x; i < kTile && f0 + i < n_out; i += kThreads) {
            OUT v = OUT(0);
            if (i < nf) {
                if constexpr (sizeof(OUT) == 2) v = frame_i16(bytes + i * block, c.format);
                else v = frame_f32(bytes + i * block, c.format, c.channels);
            }
            row[f0 + i] = v;
        }
        __syncthreads();
    }
}
#endif

}  // namespace pcm
}  // namespace b200aa
