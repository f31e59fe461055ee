// Frame and row arithmetic of feature_extraction(), spectrogram() and chromagram() for one clip of n samples (reference
// ShortTermFeatures.py:608, :413-415 and :347-355): how many frames, how many rows the output has, which of them the reference's loop fills from full frames or from a frame
// clipped at the end of the clip, and whether the single-clip entry points refuse the clip.  The host entry points, the
// row kernels of a ragged batch, the clipped-frame kernel and b200aa_row_counts all use these, so the rule lives in one
// place.  __host__ __device__: tests/rows_host.cu runs the same code on the CPU.
#pragma once
#include <cstdint>

namespace b200aa {
namespace rows {

struct Rows {
    int64_t R;          // rows of the output: np.zeros((int((n - w) / s) + 1, ...)) (:413) / int((n - s - w) / s) + 1 (:347)
    int64_t n_it;       // rows the reference's loop fills (:415 / :349); rows [n_it, R) stay zero
    int64_t n_full;     // rows whose frame has all w samples; chromagram rows [n_full, n_it) transform a clipped frame
    bool refused;       // b200aa_spectrogram / b200aa_chromagram return an error for a clip of this length
};

__host__ __device__ inline int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }

// len(range(a, b, s)) for s > 0
__host__ __device__ inline int64_t range_len(int64_t a, int64_t b, int64_t s) { return b > a ? (b - a + s - 1) / s : 0; }

// frames of feature_extraction's loop (:608): b200aa_num_frames, and the per-clip count of a ragged batch on the device
__host__ __device__ inline int64_t frames(int64_t n, int w, int s) { return n < w ? 0 : (n - w) / s + 1; }

// first sample of row i: both loops start at cur_p = w (:415, :349)
__host__ __device__ inline int64_t frame_start(int w, int s, int64_t i) { return int64_t(w) + i * s; }

// C division truncates toward zero like Python's int(x / y) on the reference's float quotient.  Every frame of the
// spectrogram's loop is full (range(w, n - w + 1, s)).  R <= 0 makes np.zeros raise; so does the normalisation of an
// empty clip (the max of no samples), which matters where s > w: there int(-w / s) + 1 = 1 row at n = 0.
__host__ __device__ inline Rows spectrogram(int64_t n, int w, int s)
{
    Rows r;
    r.R = (n - w) / s + 1;
    r.n_it = r.R > 0 ? min64(r.R, range_len(w, n - w + 1, s)) : 0;
    r.n_full = r.n_it;
    r.refused = r.R <= 0 || n == 0;
    return r;
}

// The loop range(w, n - s, s) also transforms frames clipped at the end of the clip: row i >= n_full holds the
// n - frame_start(i) < w samples left.  Refused: no rows, a clip shorter than w + s, and a clipped frame of fewer than
// K = w / 2 samples, where the reference's chroma scatter raises (the shortest clipped frame is the last one).
__host__ __device__ inline Rows chromagram(int64_t n, int w, int s)
{
    Rows r;
    r.R = (n - s - w) / s + 1;
    r.n_it = r.R > 0 ? min64(r.R, range_len(w, n - s, s)) : 0;
    r.n_full = n >= 2 * int64_t(w) ? min64(r.n_it, (n - 2 * int64_t(w)) / s + 1) : 0;
    r.refused = r.R <= 0 || n - s - w < 0 || (r.n_it > r.n_full && n - frame_start(w, s, r.n_it - 1) < w / 2);
    return r;
}

// most clipped frames a clip can have: their starts p = w + i*s satisfy n - w < p < n - s, an open interval of length
// w - s, which holds at most ceil((w - s) / s) = (w - 1) / s of them
__host__ __device__ inline int64_t max_clipped(int w, int s) { return w > s ? (int64_t(w) - 1) / s : 0; }

// mid-term windows of a clip of n_frames frames: b200aa_mid_windows on the host, per clip of a ragged batch on the device
__host__ __device__ inline int64_t windows_of(int64_t n_frames, int stepr)
{
    return (stepr < 1 || n_frames <= 0) ? 0 : (n_frames + stepr - 1) / stepr;
}

}  // namespace rows
}  // namespace b200aa
