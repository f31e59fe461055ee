// libb200aa.so -- Beat extraction (kernel 4).
#include <algorithm>
#include <cmath>

#include "../../include/b200aa.h"
#include "beat.cuh"
#include "entry.h"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 4: beat extraction (MidTermFeatures.py:18-84), bit for bit the host beat_extraction (csrc/beat.cuh)
// ------------------------------------------------------------------------------------------------
// One CTA of P = blockDim.x threads (a power of two, 32 .. 256) per (clip, beat row): threshold, chunked peak scan, and the
// distances between successive peaks counted into the row's integer histogram counts[row][d - 1], d = 1 .. min(mbt, T - 1).
// The rows are float32 (b200aa_beat_extraction) or float64 (b200aa_beat_extraction_f64); both are read as double.
template <class Real>
__device__ __forceinline__ void beat_rows(const Real *st, int F, int64_t n_frames, int64_t t_stride, const int64_t *frames,
                                          int64_t b0, int64_t mbt, int nb, int chunk, int nch_max, beat::Chunk *recs,
                                          unsigned *counts)
{
    __shared__ double part[256];
    const int64_t bl = blockIdx.x / beat::kRows;
    const int r = int(blockIdx.x - bl * beat::kRows);
    const int64_t b = b0 + bl;
    const int64_t T = frames ? min(max(frames[b], int64_t(0)), n_frames) : n_frames;
    const Real *row = st + (size_t(b) * F + beat::row_index(r)) * t_stride;
    const int P = blockDim.x, k = threadIdx.x;
    auto v = [row](int64_t i) { return double(row[i]); };
    auto absdiff = [row](int64_t i) { return fabs(beat::dsub(double(row[i]), double(row[i + 1]))); };

    const int64_t n = T > 1 ? T - 1 : 0;
    int64_t off, len;
    beat::pairwise_part(n, __ffs(P) - 1, k, off, len);
    part[k] = beat::pairwise_sum(absdiff, off, len, n);
    __syncthreads();
    for (int s = 1; s < P; s <<= 1) {
        if ((k & (2 * s - 1)) == 0) part[k] = beat::dadd(part[k], part[k + s]);
        __syncthreads();
    }
    const double delta = beat::threshold(part[0], T);

    const int32_t nch = int32_t((T + chunk - 1) / chunk);
    beat::Chunk *rec = recs + (size_t(bl) * beat::kRows + r) * nch_max;
    if (nch > 1) {
        for (int32_t c = k; c < nch; c += P)                                 // speculative pass, every chunk from the fresh state
            rec[c] = beat::spec_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta);
        __syncthreads();
        if (k == 0) {                                                         // fix-up, serial over the chunks
            beat::State s = rec[0].s;
            int32_t last = rec[0].last;
            for (int32_t c = 1; c < nch; ++c) {
                const beat::Chunk spec = rec[c];
                rec[c].s = s;
                rec[c].last = last;
                beat::fixup_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta, spec, s, last);
            }
        }
        __syncthreads();
    }
    unsigned *cnt = counts + (size_t(bl) * beat::kRows + r) * nb;
    for (int32_t c = k; c < nch; c += P) {                                    // counting pass from the true entry states
        int32_t last = c ? rec[c].last : -1;
        beat::scan_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta, c ? rec[c].s : beat::fresh(),
                         [&](int32_t p) {
                             if (last >= 0 && p - last >= 1 && p - last <= mbt) atomicAdd(cnt + (p - last - 1), 1u);
                             last = p;
                         });
    }
}
__global__ void __launch_bounds__(256) beat_rows_kernel(const float *st, int F, int64_t n_frames, int64_t t_stride,
                                                        const int64_t *frames, int64_t b0, int64_t mbt, int nb, int chunk,
                                                        int nch_max, beat::Chunk *recs, unsigned *counts)
{
    beat_rows(st, F, n_frames, t_stride, frames, b0, mbt, nb, chunk, nch_max, recs, counts);
}
__global__ void __launch_bounds__(256) beat_rows_f64_kernel(const double *st, int F, int64_t n_frames, int64_t t_stride,
                                                            const int64_t *frames, int64_t b0, int64_t mbt, int nb, int chunk,
                                                            int nch_max, beat::Chunk *recs, unsigned *counts)
{
    beat_rows(st, F, n_frames, t_stride, frames, b0, mbt, nb, chunk, nch_max, recs, counts);
}

// One warp per clip: hist[k] = sum over the rows, in _BEAT_ROWS order, of counts[row][k] / T; its first maximum k, and its
// pairwise sum over all mbt bins (bins >= nb are zero).  d_out[b] = (60 / ((k + 1) * window), hist[k] / (sum + 1e-8)).
__global__ void __launch_bounds__(256) beat_finish_kernel(const int64_t *frames, int64_t n_frames, int64_t b0, int64_t n_slice,
                                                          double window, int64_t mbt, int nb, const unsigned *counts, double *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t bl = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (bl >= n_slice) return;
    const int64_t b = b0 + bl;
    const int64_t T = frames ? min(max(frames[b], int64_t(0)), n_frames) : n_frames;
    if (T == 0) {               // every bin is 0 / 0: np.argmax picks the first NaN, the ratio is NaN
        if (lane == 0) {
            out[2 * b] = beat::ddiv(60.0, beat::dmul(1.0, window));
            out[2 * b + 1] = __longlong_as_double(0x7ff8000000000000LL);
        }
        return;
    }
    const unsigned *cnt = counts + size_t(bl) * beat::kRows * nb;
    const double Td = double(T);
    auto hist = [cnt, nb, Td](int64_t k) {
        double h = 0.0;
        for (int r = 0; r < beat::kRows; ++r) h = beat::dadd(h, beat::ddiv(double(cnt[size_t(r) * nb + k]), Td));
        return h;
    };
    double bv = 0.0;            // every bin is >= 0: (0.0, 0) is the answer when all are zero
    int64_t bk = 0;
    for (int64_t k = lane; k < nb; k += 32) {
        const double h = hist(k);
        if (h > bv) { bv = h; bk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int64_t ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov > bv || (ov == bv && ok < bk)) { bv = ov; bk = ok; }
    }
    int64_t off, len;
    beat::pairwise_part(mbt, 5, lane, off, len);
    double s = beat::pairwise_sum(hist, off, len, nb);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_down_sync(0xffffffffu, s, o);
        if ((lane & (2 * o - 1)) == 0) s = beat::dadd(s, t);
    }
    if (lane == 0) {
        out[2 * b] = beat::ddiv(60.0, beat::dmul(double(bk + 1), window));
        out[2 * b + 1] = beat::ddiv(bv, beat::dadd(s, 0.00000001));
    }
}

// b200aa_beat_extraction and b200aa_beat_extraction_f64: `rows` is the row kernel of the rows' element type
template <class Real, class RowsKernel>
static int beat_launch(RowsKernel rows, const Real *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                       const int64_t *d_frames, double window_size, double *d_out, void *stream)
{
    if (!d_st || !d_out || n_clips < 0 || n_feats < 19 || n_frames < 0 || n_frames > INT32_MAX - beat::kChunk ||
        t_stride < n_frames)
        return B200AA_ERR_INVALID;
    const double mbt_d = std::nearbyint(2.0 / window_size);               // Python's round(): half to even
    if (!(mbt_d >= 1.0) || mbt_d > double(INT32_MAX)) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t mbt = int64_t(mbt_d);
    const int nb = int(std::min<int64_t>(mbt, std::max<int64_t>(n_frames - 1, 0)));
    const int chunk = beat::kChunk;
    const int nch_max = int(std::max<int64_t>(1, (n_frames + chunk - 1) / chunk));
    int P = 32;
    while (P < nch_max && P < 256) P <<= 1;
    // scratch per clip: the rows' histograms and, for rows of more than one chunk, their chunk records; clips go in slices
    // whose scratch stays below 256 MiB
    const size_t rec_bytes = nch_max > 1 ? size_t(nch_max) * sizeof(beat::Chunk) : 0;
    const size_t per_clip = size_t(beat::kRows) * (size_t(nb) * sizeof(unsigned) + rec_bytes);
    const int64_t slice = std::max<int64_t>(1, std::min<int64_t>({n_clips, int64_t(kScratchSliceBytes / std::max<size_t>(per_clip, 1)),
                                                                   int64_t(INT32_MAX / beat::kRows)}));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(size_t(slice) * per_clip);
    if (rc != B200AA_OK) return rc;
    unsigned *counts = static_cast<unsigned *>(scratch.get());
    beat::Chunk *recs = reinterpret_cast<beat::Chunk *>(static_cast<char *>(scratch.get()) + size_t(slice) * beat::kRows * nb * sizeof(unsigned));
    for (int64_t b0 = 0; b0 < n_clips; b0 += slice) {
        const int64_t ns = std::min<int64_t>(slice, n_clips - b0);
        const cudaError_t e = nb ? cudaMemsetAsync(counts, 0, size_t(ns) * beat::kRows * nb * sizeof(unsigned), st) : cudaSuccess;
        if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync");
        rows<<<(unsigned)(ns * beat::kRows), P, 0, st>>>(d_st, n_feats, n_frames, t_stride, d_frames, b0, mbt, nb, chunk,
                                                         nch_max, recs, counts);
        CK_LAUNCH("beat_rows_kernel");
        beat_finish_kernel<<<(unsigned)((ns * 32 + 255) / 256), 256, 0, st>>>(d_frames, n_frames, b0, ns, window_size, mbt, nb,
                                                                               counts, d_out);
        CK_LAUNCH("beat_finish_kernel");
    }
    return scratch.done(B200AA_OK);
}

extern "C" int b200aa_beat_extraction(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                                      const int64_t *d_frames, double window_size, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_beat_extraction");
    return beat_launch(beat_rows_kernel, d_st, n_clips, n_feats, n_frames, t_stride, d_frames, window_size, d_out, stream);
}

extern "C" int b200aa_beat_extraction_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t n_frames,
                                          int64_t t_stride, const int64_t *d_frames, double window_size, double *d_out,
                                          void *stream)
{
    NvtxRange nvtx_("b200aa_beat_extraction_f64");
    return beat_launch(beat_rows_f64_kernel, d_st, n_clips, n_feats, n_frames, t_stride, d_frames, window_size, d_out, stream);
}
