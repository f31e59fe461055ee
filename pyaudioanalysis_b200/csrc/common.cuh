// Shared device helpers and parameter blocks for the short-term feature kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/b200aa.h"
#include "rows.cuh"

#define B200AA_EPS 2.220446049250313e-16f   /* sys.float_info.epsilon, ShortTermFeatures.py:11 */

namespace b200aa {

constexpr int kThreads = 256;       // 8 warps per CTA
constexpr int kWarps = kThreads / 32;
constexpr int kFvStride = 36;       // 34 base features per frame, padded
constexpr int kMaxRadix = 24;

// layout of the small-table blob (int32 words), copied to shared memory by every CTA
struct BlobLayout {
    int mel_start;   // [40] first bin of each filter
    int mel_count;   // [40] number of taps
    int mel_off;     // [40] offset of the first tap weight
    int mel_w;       // [mel_nnz] tap weights (float)
    int dct;         // [13 x 41] DCT rows, padded stride 41 (float)
    int chr_off;     // [13] per pitch class: first entry
    int chr_bin;     // [chr_nnz] source bin
    int chr_w;       // [chr_nnz] weight (float)
    int mel_grp;     // [16 x 3] filters in 16 groups of balanced tap count (-1 = empty slot)
    int words;       // total
};

enum Mode { kModeFeatures = 0, kModeSpectrogram = 1, kModeChromagram = 2 };

struct StParams {
    const void *sig;
    const int64_t *len;             // nullable ragged lengths
    const b200aa_clip_norm *norm;
    float *out;
    const float2 *tw;               // exp(-2 pi i j / Nc), j < Nc
    const float2 *tw_post;          // exp(-2 pi i k / N),  k < K   (packed real transform)
    const int *blob;
    BlobLayout bl;
    int64_t n_clips, n_samples, clip_stride, t_stride;
    int64_t seg_len, segs_per_clip, n_items;
    // spectrogram / chromagram launches: rows [0, rows_launch) of every clip, row r the full frame that starts at
    // rows::frame_start(window, step, r), stored at output row b * rows_launch + r; rows >= rows_valid are written as
    // zeros (the reference leaves them unset, ShortTermFeatures.py:413-422).  Frames clipped at the end of a clip
    // (:352-355) go to clipped_chroma_kernel.  A ragged row launch (len set, the kernels' RAGGED form) takes both counts
    // of clip b from ragged_rows below.
    int64_t rows_launch, rows_valid;
    int dtype, deltas, n_out;       // n_out = 34 or 68
    int window;                     // samples per frame
    int G;                          // frames per group (generic kernel)
    int step, K, Kp, Nc, packed;    // K = window/2 bins kept; Nc = complex transform length
    int nrad;
    int radix[kMaxRadix];
    // large windows (generic kernel, BIG form): the transform ping-pong buffers and the |X| rows of every CTA live in
    // global memory (stream-ordered allocation per launch) instead of shared memory
    unsigned char *scratch;
    size_t scratch_stride;          // bytes per CTA
};

// first sample of frame r: feature frames start at r * step (ShortTermFeatures.py:608), spectrogram / chromagram rows at
// rows::frame_start
template <int MODE>
__device__ __forceinline__ int64_t frame_first(int w, int s, int64_t r)
{
    return MODE == kModeFeatures ? r * s : rows::frame_start(w, s, r);
}

// Length of clip b of a ragged batch, clamped to the batch width (the clips' samples end there)
__device__ __forceinline__ int64_t ragged_len(const StParams &p, int64_t b)
{
    const int64_t n = p.len[b];
    return n < 0 ? 0 : (n > p.n_samples ? p.n_samples : n);
}

// Rows of clip b in a ragged spectrogram / chromagram launch: its own R_b (none when the single-clip entry point refuses
// the clip), of which the first n_full come from full frames; rows [n_full, R_b) are written as zeros, rows >= R_b not
// at all.  The launch itself is sized by the batch width, whose row count bounds every clip's.
template <int MODE>
__device__ __forceinline__ void ragged_rows(const StParams &p, int64_t b, int64_t &n_rows, int64_t &n_valid)
{
    const int64_t n = ragged_len(p, b);
    const rows::Rows r = MODE == kModeSpectrogram ? rows::spectrogram(n, p.window, p.step) : rows::chromagram(n, p.window, p.step);
    n_rows = r.refused ? 0 : r.R;
    n_valid = r.refused ? 0 : r.n_full;
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ int warp_min_int(int v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b)
{
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}

// sample -> float, minus the clip's exact-in-float centre m (see b200aa_clip_norm)
struct SampleReader {
    const void *base;   // first sample of the clip
    int dtype;
    float m;
    __device__ __forceinline__ float operator()(int64_t n) const
    {
        float v = dtype == B200AA_DTYPE_I16 ? float(reinterpret_cast<const short *>(base)[n])
                                            : reinterpret_cast<const float *>(base)[n];
        return v - m;
    }
};

// ----------------------------------------------------------------------------------------
// Per-frame features, one warp per frame.  X = |FFT|[0:K]/K of this frame in shared memory,
// Xp = the previous frame's (or X itself for the first frame), sx / sxp = their plain sums.
// Writes 34 values to fv (shared).  Reference lines: see each block.
// ----------------------------------------------------------------------------------------
struct SmallTables {
    const int *mel_start, *mel_count, *mel_off;
    const float *mel_w, *dct;
    const int *chr_off, *chr_bin;
    const float *chr_w;
};

__device__ __forceinline__ SmallTables bind_tables(const int *blob_s, const BlobLayout &bl)
{
    SmallTables t;
    t.mel_start = blob_s + bl.mel_start;
    t.mel_count = blob_s + bl.mel_count;
    t.mel_off = blob_s + bl.mel_off;
    t.mel_w = reinterpret_cast<const float *>(blob_s + bl.mel_w);
    t.dct = reinterpret_cast<const float *>(blob_s + bl.dct);
    t.chr_off = blob_s + bl.chr_off;
    t.chr_bin = blob_s + bl.chr_bin;
    t.chr_w = reinterpret_cast<const float *>(blob_s + bl.chr_w);
    return t;
}

// chroma vector (12 lanes) from X: (M @ X^2) / sum(X^2)   [ShortTermFeatures.py:285-308]
__device__ __forceinline__ float chroma_lane(const float *X, float sxx, const SmallTables &tb, int lane)
{
    float acc = 0.f;
    if (lane < 12) {
        const int e0 = tb.chr_off[lane], e1 = tb.chr_off[lane + 1];
        for (int e = e0; e < e1; ++e) {
            const float v = X[tb.chr_bin[e]];
            acc = fmaf(v * v, tb.chr_w[e], acc);
        }
        acc = acc / (sxx == 0.f ? B200AA_EPS : sxx);
    }
    return acc;
}

// spectral half of the feature vector: rows 3..7, 8..20, 21..33
__device__ __forceinline__ void spectral_features(const float *X, const float *Xp, float sxp, int K,
                                                  const SmallTables &tb, float *mscratch, float *fv, int lane,
                                                  float *sx_out)
{
    // pass 1: sums  [spectral_centroid_spread :57-82, spectral_flux sums :118-119]
    float sx = 0.f, sk = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float v = X[k];
        sx += v;
        sk = fmaf(float(k + 1), v, sk);
    }
    sx = warp_sum(sx);
    sk = warp_sum(sk);
    const float invK = 1.f / float(K);
    // centroid / spread, already divided by fs/2:  ind_k / (fs/2) = (k+1)/K.
    // Xt = X / max(X) only rescales numerator and denominator; DEN = sum(Xt)+eps >= 1 so eps is
    // below float resolution.  max == 0  <=>  sx == 0  ->  the reference gets 0 for both.
    float cen = 0.f, spr = 0.f;
    if (sx > 0.f) cen = (sk / sx) * invK;
    // pass 2: spread, flux, spectral-entropy blocks, rolloff
    float sp = 0.f, fl = 0.f;
    const float nx = 1.f / (sx + float(K) * B200AA_EPS);
    const float np_ = 1.f / (sxp + float(K) * B200AA_EPS);
    for (int k = lane; k < K; k += 32) {
        const float v = X[k];
        const float d = float(k + 1) * invK - cen;
        sp = fmaf(d * d, v, sp);
        const float df = v * nx - Xp[k] * np_;
        fl = fmaf(df, df, fl);
    }
    sp = warp_sum(sp);
    fl = warp_sum(fl);
    if (sx > 0.f) spr = sqrtf(sp / sx);
    // rolloff [:127-140]: contiguous chunks per lane (odd length => conflict-free), warp scan
    int c = (K + 31) / 32;
    c |= 1;
    const int k0 = lane * c, k1 = min(K, k0 + c);
    float part = 0.f;
    for (int k = k0; k < k1; ++k) part = fmaf(X[k], X[k], part);
    float incl = part;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    const float sxx = __shfl_sync(0xffffffffu, incl, 31);
    const float thr = 0.90f * sxx;
    float run = incl - part;
    int first = 0x7fffffff;
    for (int k = k0; k < k1; ++k) {
        run = fmaf(X[k], X[k], run);
        if (first == 0x7fffffff && run + B200AA_EPS > thr) first = k;
    }
    first = warp_min_int(first);
    const float roll = first == 0x7fffffff ? 0.f : float(first) * invK;
    // spectral entropy [:85-107]: 10 blocks of floor(K/10) bins, total over all K bins
    const int Lb = K / 10;
    float ent = 0.f;
    for (int j = 0; j < 10; ++j) {
        float e = 0.f;
        for (int k = j * Lb + lane; k < (j + 1) * Lb; k += 32) e = fmaf(X[k], X[k], e);
        e = warp_sum(e);
        const float s = e / (sxx + B200AA_EPS);
        ent -= s * log2f(s + B200AA_EPS);
    }
    // mfcc [:236-254]: 40 sparse triangular filters, log10, 13 DCT rows.
    // DCT rows 1..12 are orthogonal to constants, so they are applied to (m - mean(m)): identical
    // in exact arithmetic, and it removes the float32 cancellation error when the log-mel
    // spectrum is nearly flat (digital silence: every m equals log10(eps) = -15.65).
    float msum = 0.f;
    for (int i = lane; i < B200AA_N_MEL; i += 32) {
        const int s0 = tb.mel_start[i], cnt = tb.mel_count[i], off = tb.mel_off[i];
        float acc = 0.f;
        for (int j = 0; j < cnt; ++j) acc = fmaf(X[s0 + j], tb.mel_w[off + j], acc);
        const float m = log10f(acc + B200AA_EPS);
        mscratch[i] = m;
        msum += m;
    }
    const float mbar = warp_sum(msum) * (1.f / float(B200AA_N_MEL));
    __syncwarp();
    if (lane < B200AA_N_MFCC) {
        float acc = 0.f;
        const float *row = tb.dct + lane * 41;
#pragma unroll 8
        for (int n = 0; n < B200AA_N_MEL; ++n) acc = fmaf(row[n], mscratch[n] - mbar, acc);
        fv[8 + lane] = lane == 0 ? 6.324555320336759f * mbar : acc;     // row 0: sqrt(1/40) * sum(m)
    }
    // chroma [:277-321] + population std of the 12 values [:667]
    const float ch = chroma_lane(X, sxx, tb, lane);
    const float mean = warp_sum(ch) * (1.f / 12.f);
    const float dv = lane < 12 ? ch - mean : 0.f;
    const float var = warp_sum(dv * dv) * (1.f / 12.f);
    if (lane < 12) fv[21 + lane] = ch;
    if (lane == 0) {
        fv[3] = cen;
        fv[4] = spr;
        fv[5] = ent;
        fv[6] = fl;
        fv[7] = roll;
        fv[33] = sqrtf(var);
        *sx_out = sx;
    }
    __syncwarp();
}

// sign(x - mean) in {-1, 0, +1} as a float, from the exact thresholds of b200aa_clip_norm
__device__ __forceinline__ float sign_class(float d, float lo, float hi) { return (d > lo ? 1.f : 0.f) - (d < hi ? 1.f : 0.f); }

// ---- time-domain rows: zcr, energy, energy entropy  [ShortTermFeatures.py:22-51], one warp per frame.  D(n) returns
// sample n of the frame minus the clip centre m.  Every lane owns c = ceil(w/32) CONSECUTIVE samples (one load per
// sample, sequential sign flips, energy split at the single entropy-block boundary a chunk can contain); the block
// energies are then sums of lane parts.
// Per-lane constants (depend on w and the lane only; computed once per CTA into shared memory as int4):
//   x = c, y = samples of the chunk that belong to the earlier block, [z, w) = parts that make up block `lane` (< 10)
__device__ inline int4 time_lane_init(int w, int lane)
{
    const int c = (w + 31) / 32, L = w / 10;
    const int k0 = lane * c, end = min(w, k0 + c);
    int split = 0;
    if (L > 0 && end > k0) {
        const int bnd = ((end - 1) / L) * L;
        split = bnd > k0 ? bnd - k0 : 0;
    }
    int ps = 64, pe = 0;
    if (lane < 10 && L > 0) {
        const int j = lane;
        for (int q = 0; q < 32; ++q) {
            const int b0 = q * c, e0 = min(w, b0 + c);
            if (e0 <= b0) break;
            const int bb = ((e0 - 1) / L) * L, sp = bb > b0 ? bb - b0 : 0;
            if (sp > 0 && b0 >= j * L && b0 + sp <= (j + 1) * L) { ps = min(ps, 2 * q); pe = max(pe, 2 * q + 1); }
            if (b0 + sp >= j * L && e0 <= (j + 1) * L) { ps = min(ps, 2 * q + 1); pe = max(pe, 2 * q + 2); }
        }
    }
    if (pe <= ps) { ps = 0; pe = 0; }
    return make_int4(c, split, ps, pe);
}

template <class Acc>
__device__ __forceinline__ void time_features_chunked(Acc D, int w, const b200aa_clip_norm &nm, int4 tl, float *parts,
                                                      float *fv, int lane)
{
    const float a = nm.a, bp = nm.bp, lo = nm.lo, hi = nm.hi;
    const int c = tl.x, k0 = lane * c, end = min(w, k0 + c);
    float plo = 0.f, phi = 0.f, fl = 0.f;
    float sprev = (k0 > 0 && k0 < w) ? sign_class(D(k0 - 1), lo, hi) : 0.f;
    for (int n = k0; n < end; ++n) {
        const float d = D(n);
        const float y = fmaf(a, d, bp);
        const float sq = y * y;
        if (n - k0 < tl.y) plo += sq; else phi += sq;
        const float sg = sign_class(d, lo, hi);
        if (n > 0) fl += fabsf(sg - sprev);
        sprev = sg;
    }
    parts[2 * lane] = plo;
    parts[2 * lane + 1] = phi;
    __syncwarp();
    const float tot = warp_sum(plo + phi);
    fl = warp_sum(fl);
    float e = 0.f;
    for (int q = tl.z; q < tl.w; ++q) e += parts[q];
    float H = 0.f;
    if (lane < 10) {
        const float sj = e / (tot + B200AA_EPS);
        H = -sj * log2f(sj + B200AA_EPS);
    }
    H = warp_sum(H);
    if (lane == 0) {
        fv[0] = fl * 0.5f / float(w - 1);
        fv[1] = tot / float(w);
        fv[2] = H;
    }
    __syncwarp();
}

}  // namespace b200aa
