// libb200aa.so -- Mid-term pooling (kernel 2), the long-term mean, per-clip frame / row counts and normalize_windows (kernel 3).
#include "../../include/b200aa.h"
#include "entry.h"
#include "rows.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 2: mid-term pooling (MidTermFeatures.py:110-126): one warp per (clip, feature row, window)
// ------------------------------------------------------------------------------------------------
// frames (nullable, int64 [n_clips]): clip b has T_b = clamp(frames[b], 0, t_stride) frames and M_b = windows_of(T_b)
// windows; warps of windows j >= M_b write nothing.  Without frames every clip has T frames.  A warp's sums depend only
// on (c0, c1, lane), so a clip pooled in a ragged batch gives bit for bit what it gives alone with T = T_b.  RAGGED is
// a template flag only so that the batch without counts keeps the code (and time) it had before counts existed.
template <bool RAGGED>
__global__ void __launch_bounds__(256) mid_pool_kernel(const float *st, int64_t n_clips, int F, int64_t T,
                                                        int64_t t_stride, const int64_t *frames, int ratio, int stepr,
                                                        int64_t M, float *mid)
{
    const int lane = threadIdx.x & 31;
    const int64_t wid = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t total = n_clips * F * M;
    if (wid >= total) return;
    const int64_t j = wid % M, bf = wid / M;
    const int64_t b = bf / F;
    const int f = int(bf - b * F);
    if (RAGGED) {
        T = min(max(frames[b], int64_t(0)), t_stride);
        if (j >= rows::windows_of(T, stepr)) return;              // the whole warp: j is uniform across it
    }
    // window j is the Python slice row[c0 : min(c0 + ratio, T)] (:116-120): a negative end counts from the end of
    // the row (ratio < 0), an end before c0 gives an empty window; n = 0 makes mean and std 0 / 0 -> 0 below
    const int64_t c0 = j * stepr;
    int64_t c1 = min(T, c0 + ratio);
    if (c1 < 0) c1 = max(c1 + T, int64_t(0));
    const float *row = st + (size_t(b) * F + f) * t_stride;
    const int n = int(max(c1 - c0, int64_t(0)));
    double s = 0.0;
    for (int64_t c = c0 + lane; c < c1; c += 32) s += double(row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double mean = s / double(n);
    double v = 0.0;
    for (int64_t c = c0 + lane; c < c1; c += 32) { const double d = double(row[c]) - mean; v += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) {
        float mu = float(mean), sd = float(sqrt(v / double(n)));
        // np.nan_to_num (:126)
        if (isnan(mu)) mu = 0.f;
        if (isnan(sd)) sd = 0.f;
        if (isinf(mu)) mu = mu > 0 ? 3.4028234664e38f : -3.4028234664e38f;
        if (isinf(sd)) sd = 3.4028234664e38f;
        mid[(size_t(b) * 2 * F + f) * M + j] = mu;
        mid[(size_t(b) * 2 * F + F + f) * M + j] = sd;
    }
}

// d_mid's row stride is M = windows_of(T): with frames, T = t_stride, the longest any clip can have
static int mid_pool_launch(const float *d_st, int64_t n_clips, int n_feats, int64_t T, int64_t t_stride, const int64_t *d_frames,
                           int ratio, int step_ratio, float *d_mid, void *stream)
{
    const int64_t M = rows::windows_of(T, step_ratio);
    const int64_t warps = n_clips * n_feats * M;
    if (warps == 0) return B200AA_OK;
    const int64_t blocks = (warps * 32 + 255) / 256;
    auto kernel = d_frames ? mid_pool_kernel<true> : mid_pool_kernel<false>;
    kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_st, n_clips, n_feats, T, t_stride, d_frames,
                                                                             ratio, step_ratio, M, d_mid);
    CK_LAUNCH("mid_pool_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_mid_pool(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                               int ratio, int step_ratio, float *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool");
    if (!d_st || !d_mid || n_clips < 0 || n_feats < 1 || n_frames < 1 || step_ratio < 1 || t_stride < n_frames)
        return B200AA_ERR_INVALID;
    return mid_pool_launch(d_st, n_clips, n_feats, n_frames, t_stride, nullptr, ratio, step_ratio, d_mid, stream);
}

extern "C" int b200aa_mid_pool_ragged(const float *d_st, int64_t n_clips, int n_feats, int64_t t_stride,
                                      const int64_t *d_frames, int ratio, int step_ratio, float *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool_ragged");
    if (!d_st || !d_frames || !d_mid || n_clips < 0 || n_feats < 1 || step_ratio < 1 || t_stride < 0)
        return B200AA_ERR_INVALID;
    return mid_pool_launch(d_st, n_clips, n_feats, t_stride, t_stride, d_frames, ratio, step_ratio, d_mid, stream);
}

// long-term average of the mid-term matrix: one warp per (clip, row), fp64 accumulation.  windows (nullable, int64
// [n_clips]): clip b averages its first M_b = clamp(windows[b], 0, M) columns (0 / 0 = NaN for none, as np.mean of an
// empty axis); the sum's order depends only on (M_b, lane), as in mid_pool_kernel.
__global__ void __launch_bounds__(256) long_term_mean_kernel(const float *mid, int64_t all_rows, int n_rows, int64_t M,
                                                             const int64_t *windows, float *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t wid = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (wid >= all_rows) return;
    const int64_t Mb = windows ? min(max(windows[wid / n_rows], int64_t(0)), M) : M;
    const float *row = mid + size_t(wid) * M;
    double s = 0.0;
    for (int64_t c = lane; c < Mb; c += 32) s += double(row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[wid] = float(s / double(Mb));
}

static int long_term_mean_launch(const float *d_mid, int64_t n_clips, int n_rows, int64_t m_stride, const int64_t *d_windows,
                                 float *d_out, void *stream)
{
    const int64_t rows = n_clips * n_rows;
    if (rows == 0) return B200AA_OK;
    const int64_t blocks = (rows * 32 + 255) / 256;
    long_term_mean_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_mid, rows, n_rows, m_stride,
                                                                                             d_windows, d_out);
    CK_LAUNCH("long_term_mean_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_long_term_mean(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, float *d_out, void *stream)
{
    if (!d_mid || !d_out || n_clips < 0 || n_rows < 1 || n_windows < 1) return B200AA_ERR_INVALID;
    return long_term_mean_launch(d_mid, n_clips, n_rows, n_windows, nullptr, d_out, stream);
}

extern "C" int b200aa_long_term_mean_ragged(const float *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                            const int64_t *d_windows, float *d_out, void *stream)
{
    if (!d_mid || !d_windows || !d_out || n_clips < 0 || n_rows < 1 || m_stride < 0) return B200AA_ERR_INVALID;
    return long_term_mean_launch(d_mid, n_clips, n_rows, m_stride, d_windows, d_out, stream);
}

// per-clip counts of a ragged batch from its device lengths: one thread per clip
__global__ void __launch_bounds__(256) frame_counts_kernel(const int64_t *len, int64_t n_clips, int w, int s, int stepr,
                                                           int64_t *frames, int64_t *windows)
{
    const int64_t b = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (b >= n_clips) return;
    const int64_t T = rows::frames(len[b], w, s);
    frames[b] = T;
    if (windows) windows[b] = rows::windows_of(T, stepr);
}

extern "C" int b200aa_frame_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int step_ratio,
                                   int64_t *d_frames, int64_t *d_windows, void *stream)
{
    if (!d_len || !d_frames || n_clips < 0 || window < 1 || step < 1 || (d_windows && step_ratio < 1))
        return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    const int64_t blocks = (n_clips + 255) / 256;
    frame_counts_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_len, n_clips, window, step,
                                                                                           step_ratio, d_frames, d_windows);
    CK_LAUNCH("frame_counts_kernel");
    return B200AA_OK;
}

// per-clip output rows of a ragged spectrogram (which = 0) / chromagram (1): R_b, or 0 where the single-clip entry point
// refuses the clip
__global__ void __launch_bounds__(256) row_counts_kernel(const int64_t *len, int64_t n_clips, int w, int s, int which, int64_t *out)
{
    const int64_t b = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (b >= n_clips) return;
    const rows::Rows r = which ? rows::chromagram(len[b], w, s) : rows::spectrogram(len[b], w, s);
    out[b] = r.refused ? 0 : r.R;
}

extern "C" int b200aa_row_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int which, int64_t *d_rows,
                                 void *stream)
{
    if (!d_len || !d_rows || n_clips < 0 || window < 1 || step < 1 || (which != 0 && which != 1)) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    const int64_t blocks = (n_clips + 255) / 256;
    row_counts_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_len, n_clips, window, step, which, d_rows);
    CK_LAUNCH("row_counts_kernel");
    return B200AA_OK;
}

// (mid[b, f, j] - mean[f]) / std[f] -> out[b, j, f]: 32 x 32 tiles through shared memory, both sides coalesced
// (audioSegmentation.py:581-584: one column of the mid-term matrix at a time)
__global__ void normalize_windows_kernel(const float *__restrict__ mid, int n_rows, int64_t n_windows, const float *__restrict__ mean,
                                         const float *__restrict__ sd, float *__restrict__ out)
{
    __shared__ float tile[32][33];
    const int64_t b = blockIdx.z;
    const int64_t j0 = int64_t(blockIdx.x) * 32;
    const int f0 = blockIdx.y * 32;
    const float *src = mid + b * n_rows * n_windows;
    float *dst = out + b * n_rows * n_windows;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int f = f0 + r;
        const int64_t j = j0 + threadIdx.x;
        if (f < n_rows && j < n_windows) tile[r][threadIdx.x] = (src[int64_t(f) * n_windows + j] - mean[f]) / sd[f];
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t j = j0 + r;
        const int f = f0 + threadIdx.x;
        if (f < n_rows && j < n_windows) dst[j * n_rows + f] = tile[threadIdx.x][r];
    }
}

extern "C" int b200aa_normalize_windows(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, const float *d_mean,
                                        const float *d_std, float *d_out, void *stream)
{
    if (!d_mid || !d_out || !d_mean || !d_std || n_clips < 0 || n_rows < 1 || n_windows < 0) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(stream, "b200aa_normalize_windows", "not captured; call it eagerly");
    if (n_clips == 0 || n_windows == 0) return B200AA_OK;
    if (n_clips > 65535 || (n_rows + 31) / 32 > 65535) return B200AA_ERR_UNSUPPORTED;
    const dim3 grid((unsigned)((n_windows + 31) / 32), (unsigned)((n_rows + 31) / 32), (unsigned)n_clips), block(32, 8);
    normalize_windows_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(d_mid, n_rows, n_windows, d_mean, d_std, d_out);
    CK_LAUNCH("normalize_windows_kernel");
    return B200AA_OK;
}
