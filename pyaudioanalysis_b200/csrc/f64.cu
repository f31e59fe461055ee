// libb200aa.so -- the float64 feature path (kernel family 12): clip normalisation, short-term features, spectrogram and
// chromagram rows, mid-term pooling and the long-term mean, all in float64 (csrc/f64.cuh states the arithmetic).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "../../include/b200aa.h"
#include "common.cuh"
#include "entry.h"
#include "f64.cuh"
#include "rows.cuh"
#include "tables.inl"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// a plan's float64 tables
// ------------------------------------------------------------------------------------------------
struct F64Tables {
    std::vector<int> radix;                     // the transform of length window: its Stockham radices
    b200aa_host::DeviceMemory tw;               // double2 [window]: exp(-2 pi i j / window)
    b200aa_host::DeviceMemory mel_idx;          // int [3 x 40]: first bin, taps, offset of the first weight of each filter
    b200aa_host::DeviceMemory mel_w;            // double [taps]
    b200aa_host::DeviceMemory dct;              // double [13 x 40]
    b200aa_host::DeviceMemory chr_idx;          // int [13 + entries]: per pitch class the first entry, then each entry's bin
    b200aa_host::DeviceMemory chr_div;          // double [entries]: share[semis[j]] of each entry's slot j
};

// The chroma scatter of the loop flavour (oracle._chroma_frame): slot j of C holds spec[winner[j]] / share[semis[j]]
// (winner[j] the last bin k with semis[k] == j, negative slots wrapping), and pitch class c adds the slots j = c (mod 12)
// in ascending order.  Slots without a winner hold 0 and are left out.
static void chroma_entries(int fs, int K, std::vector<int> &idx, std::vector<double> &div)
{
    std::vector<long> semi;
    std::vector<double> share;
    b200aa_host::chroma_index(fs, K, semi, share);
    auto wrap = [K](long j) -> long { return j < 0 ? j + K : j; };
    std::vector<long> winner(K, -1);
    for (int k = 0; k < K; ++k) winner[wrap(semi[k])] = k;
    std::vector<int> bins;
    idx.assign(13, 0);
    div.clear();
    for (int c = 0; c < 12; ++c) {
        idx[c] = int(bins.size());
        for (int j = c; j < K; j += 12)
            if (winner[j] >= 0) {
                bins.push_back(int(winner[j]));
                div.push_back(share[wrap(semi[j])]);
            }
    }
    idx[12] = int(bins.size());
    idx.insert(idx.end(), bins.begin(), bins.end());
    if (div.empty()) div.push_back(0.0);        // a valid allocation
}

int f64_tables_build(int fs, int window, int tables_status, std::shared_ptr<const F64Tables> &out)
{
    auto t = std::make_shared<F64Tables>();
    const int K = window / 2;
    t->radix = b200aa_host::radix_list(window);
    if (window == 1) t->radix.clear();
    if (int(t->radix.size()) > kMaxRadix) return B200AA_ERR_UNSUPPORTED;
    std::vector<double> tw(size_t(2) * window);
    for (int j = 0; j < window; ++j) {
        const double a = -2.0 * b200aa_host::kPi * double(j) / double(window);
        tw[2 * j] = std::cos(a);
        tw[2 * j + 1] = std::sin(a);
    }
    CK(b200aa_host::upload(tw, t->tw));
    std::vector<int> mel_idx(3 * 40, 0);
    std::vector<double> mel_w(1, 0.0), dct;
    std::vector<int> chr_idx(13, 0);
    std::vector<double> chr_div(1, 0.0);
    if (tables_status == B200AA_OK) {           // the tables feature_extraction and chromagram need
        std::vector<double> mel;
        b200aa_host::build_mel(fs, K, mel);
        mel_w.clear();
        for (int i = 0; i < 40; ++i) {
            int lo = -1, hi = -1;
            for (int k = 0; k < K; ++k)
                if (mel[size_t(i) * K + k] != 0.0) { if (lo < 0) lo = k; hi = k; }
            mel_idx[80 + i] = int(mel_w.size());
            if (lo >= 0) {
                mel_idx[i] = lo;
                mel_idx[40 + i] = hi - lo + 1;
                for (int k = lo; k <= hi; ++k) mel_w.push_back(mel[size_t(i) * K + k]);
            }
        }
        if (mel_w.empty()) mel_w.push_back(0.0);
        chroma_entries(fs, K, chr_idx, chr_div);
    }
    b200aa_host::build_dct(dct);
    CK(b200aa_host::upload(mel_idx, t->mel_idx));
    CK(b200aa_host::upload(mel_w, t->mel_w));
    CK(b200aa_host::upload(dct, t->dct));
    CK(b200aa_host::upload(chr_idx, t->chr_idx));
    CK(b200aa_host::upload(chr_div, t->chr_div));
    out = std::move(t);
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel 12a: clip normalisation, one warp per clip
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sample_at(const void *clip, int dtype, int64_t i)
{
    if (dtype == B200AA_DTYPE_I16) return double(static_cast<const short *>(clip)[i]);
    if (dtype == B200AA_DTYPE_F32) return double(static_cast<const float *>(clip)[i]);
    return static_cast<const double *>(clip)[i];
}
__host__ __device__ inline size_t sample_bytes(int dtype) { return dtype == B200AA_DTYPE_I16 ? 2 : dtype == B200AA_DTYPE_F32 ? 4 : 8; }

// NumPy's pairwise sum of get(0 .. n - 1), every lane of the warp taking its part (f64::lane_pairwise) and the parts
// combined in tree order: at step o, lane k (a multiple of 2o) adds lane k + o's subtree; every lane returns the total
template <class G>
__device__ double warp_np_sum(const G &get, int64_t n, int lane)
{
    double s = f64::lane_pairwise(get, n, f64::kLevels, lane);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_down_sync(0xffffffffu, s, o);
        s = npy::dadd(s, t);
    }
    return npy::dadd(0.0, __shfl_sync(0xffffffffu, s, 0));
}

__device__ __forceinline__ double warp_max_d(double v)      // NaN wins, as in np.max
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double t = __shfl_xor_sync(0xffffffffu, v, o);
        v = (t > v || t != t) ? t : v;
    }
    return v;
}

__device__ __forceinline__ int64_t clip_len(const int64_t *len, int64_t b, int64_t n_samples)
{
    if (!len) return n_samples;
    const int64_t n = len[b];
    return n < 0 ? 0 : (n > n_samples ? n_samples : n);
}

__global__ void __launch_bounds__(256) f64_norm_kernel(const void *sig, int dtype, int64_t n_clips, int64_t n_samples,
                                                       int64_t clip_stride, const int64_t *len, b200aa_clip_norm_f64 *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t b = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (b >= n_clips) return;
    const int64_t L = clip_len(len, b, n_samples);
    const void *clip = static_cast<const char *>(sig) + size_t(b) * clip_stride * sample_bytes(dtype);
    if (L == 0) {                   // no frames read the record; the reference refuses an empty clip
        if (lane == 0) out[b] = b200aa_clip_norm_f64{0.0, 1e-10};
        return;
    }
    const double s = warp_np_sum([&](int64_t i) { return f64::scaled(sample_at(clip, dtype, i)); }, L, lane);
    const double mean = npy::ddiv(s, double(L));
    double mx = 0.0;
    for (int64_t i = lane; i < L; i += 32) {
        const double v = fabs(npy::dsub(f64::scaled(sample_at(clip, dtype, i)), mean));
        mx = (v > mx || v != v) ? v : mx;
    }
    mx = warp_max_d(mx);
    if (lane == 0) out[b] = b200aa_clip_norm_f64{mean, npy::dadd(mx, 1e-10)};
}

extern "C" int b200aa_clip_stats_f64(const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples, int64_t clip_stride,
                                    const int64_t *d_len, b200aa_clip_norm_f64 *d_norm, void *stream)
{
    NvtxRange nvtx_("b200aa_clip_stats_f64");
    if (!d_sig || !d_norm || n_clips < 0 || n_samples < 0 || clip_stride < n_samples ||
        (dtype != B200AA_DTYPE_I16 && dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    const int64_t blocks = (n_clips * 32 + 255) / 256;
    f64_norm_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_sig, dtype, n_clips, n_samples,
                                                                                      clip_stride, d_len, d_norm);
    CK_LAUNCH("f64_norm_kernel");
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel 12b: frames, one warp (one CTA) per segment of consecutive frames or rows of a clip
// ------------------------------------------------------------------------------------------------
struct F64Params {
    const void *sig;
    const int64_t *len;
    const b200aa_clip_norm_f64 *norm;
    double *out;
    const double2 *tw;
    const int *mel_idx, *chr_idx;
    const double *mel_w, *dct, *chr_div;
    int64_t n_clips, n_samples, clip_stride, t_stride;
    int64_t rows_launch, seg_len, segs_per_clip, n_items;
    int dtype, fs, window, step, K, n_out;
    int nrad;
    int radix[kMaxRadix];
    unsigned char *scratch;                     // BIG: every CTA's arrays in global memory, warp_bytes apart
    size_t warp_bytes;
};

// bytes of one warp's arrays: two complex buffers of the window and two |X| rows
// (at least 20 entries each: the free one holds the 40 log-mel values of a frame)
__host__ __device__ inline int f64_buf_len(int w) { return w < 20 ? 20 : w; }
__host__ __device__ inline size_t f64_warp_bytes(int w, int K)
{
    return (size_t(f64_buf_len(w)) * 2 * sizeof(double2) + size_t(K) * 2 * sizeof(double) + 15) & ~size_t(15);
}

// |X|[0:K] / K of the frame of n samples at s0 (n = window: the plan's transform; n < window: a clipped chromagram frame,
// transformed directly over a table of its n twiddles) into X.  A and B: the warp's complex buffers.  With `time`, rows
// 0-2 of the frame go to time[0..2] first.  Returns the buffer that is free afterwards.
__device__ double2 *f64_spectrum(const F64Params &p, const void *clip, const b200aa_clip_norm_f64 &nm, int64_t s0, int n,
                                 double2 *A, double2 *B, double *X, double *time, int lane)
{
    const int w = p.window, K = p.K;
    for (int i = lane; i < n; i += 32) A[i] = make_double2(f64::normalised(sample_at(clip, p.dtype, s0 + i), nm), 0.0);
    __syncwarp();
    if (time) {
        // zcr (:22-26): the integer sum of |sign(x[i]) - sign(x[i - 1])|; energy (:29-31); energy entropy (:34-51)
        int flips = 0;
        for (int i = lane + 1; i < n; i += 32) flips += abs(f64::sign_of(A[i].x) - f64::sign_of(A[i - 1].x));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) flips += __shfl_xor_sync(0xffffffffu, flips, o);
        const double tot = warp_np_sum([A](int64_t i) { return npy::dmul(A[i].x, A[i].x); }, n, lane);
        const int blk = n / 10;
        double t = 0.0;
        if (lane < 10) {
            const double *base = &A[lane * blk].x;
            const double e = front::np_sum([base](int64_t i) { const double v = base[2 * i]; return npy::dmul(v, v); }, blk, true);
            t = f64::entropy_term(e, tot, [](double v) { return log2(v); });
        }
        double terms[10];
#pragma unroll
        for (int j = 0; j < 10; ++j) terms[j] = __shfl_sync(0xffffffffu, t, j);
        if (lane == 0) {
            time[0] = f64::zcr_of(flips, n);
            time[1] = f64::energy_of(tot, n);
            time[2] = f64::entropy_of(terms);
        }
    }
    if (n == w) {
        double2 *src = A, *dst = B;
        int Ns = 1;
        for (int ps = 0; ps < p.nrad; ++ps) {
            const int R = p.radix[ps];
            for (int o = lane; o < w; o += 32) {
                const f64::Cplx z = f64::stockham_output([src](int i) { return f64::Cplx{src[i].x, src[i].y}; }, o, w, Ns, R,
                                                         [&p](int i) { const double2 t = __ldg(p.tw + i); return f64::Cplx{t.x, t.y}; });
                dst[o] = make_double2(z.x, z.y);
            }
            __syncwarp();
            double2 *t_ = src; src = dst; dst = t_;
            Ns *= R;
        }
        for (int k = lane; k < K; k += 32) X[k] = f64::magnitude(f64::Cplx{src[k].x, src[k].y}, K);
        __syncwarp();
        return dst;
    }
    // clipped frame: X[k] = sum_j z[j] W_n^(j k mod n)
    for (int j = lane; j < n; j += 32) {
        double sn, cs;
        sincospi(2.0 * double(j) / double(n), &sn, &cs);
        B[j] = make_double2(cs, -sn);
    }
    __syncwarp();
    for (int k = lane; k < K; k += 32) {
        double re = 0.0, im = 0.0;
        int ph = 0;
        for (int j = 0; j < n; ++j) {
            const double2 t = B[ph];
            re = fma(A[j].x, t.x, re);
            im = fma(A[j].x, t.y, im);
            ph += k;
            if (ph >= n) ph -= n;
        }
        X[k] = f64::magnitude(f64::Cplx{re, im}, K);
    }
    __syncwarp();
    return B;
}

// sum(X^2) of a row, shared by the spectral entropy, the rolloff and the chroma (np.sum of the same array each time)
__device__ __forceinline__ double sum_sq(const double *X, int K, int lane)
{
    return warp_np_sum([X](int64_t k) { return npy::dmul(X[k], X[k]); }, K, lane);
}

// the chroma vector of X (:277-321, the loop flavour): lanes 0..11 return their pitch class's value
__device__ __forceinline__ double f64_chroma(const F64Params &p, const double *X, double tot, int lane)
{
    double acc = 0.0;
    if (lane < 12) {
        const int *bins = p.chr_idx + 13;
        for (int e = p.chr_idx[lane]; e < p.chr_idx[lane + 1]; ++e)
            acc = npy::dadd(acc, npy::ddiv(npy::dmul(X[bins[e]], X[bins[e]]), p.chr_div[e]));
        acc = npy::ddiv(acc, tot == 0.0 ? f64::kEps : tot);
    }
    return acc;
}

// rows 3..33 of a frame from X and the previous frame's Xp (:57-321), written to out[f * t_stride]; `scr` holds 40 doubles
__device__ void f64_spectral(const F64Params &p, const double *X, const double *Xp, double *scr, double *out, int lane)
{
    const int K = p.K;
    const double fs = double(p.fs), EPS = f64::kEps;
    // centroid and spread (:57-82)
    double top = 0.0;
    for (int k = lane; k < K; k += 32) top = fmax(top, X[k]);
    top = warp_max_d(top);
    const double dv = top == 0.0 ? EPS : top;
    const double step_hz = npy::ddiv(fs, npy::dmul(2.0, double(K)));
    const double den = npy::dadd(warp_np_sum([X, dv](int64_t k) { return npy::ddiv(X[k], dv); }, K, lane), EPS);
    const double cen = npy::ddiv(warp_np_sum([X, dv, step_hz](int64_t k) { return npy::dmul(npy::dmul(double(k + 1), step_hz), npy::ddiv(X[k], dv)); }, K, lane), den);
    const double spr = npy::dsqrt(npy::ddiv(warp_np_sum([X, dv, step_hz, cen](int64_t k) {
        const double d = npy::dsub(npy::dmul(double(k + 1), step_hz), cen);
        return npy::dmul(npy::dmul(d, d), npy::ddiv(X[k], dv));
    }, K, lane), den));
    // spectral entropy (:85-107)
    const double tot = sum_sq(X, K, lane);
    const int blk = K / 10;
    double t = 0.0;
    if (lane < 10) {
        const double *base = X + lane * blk;
        const double e = front::np_sum([base](int64_t i) { return npy::dmul(base[i], base[i]); }, blk, true);
        t = f64::entropy_term(e, tot, [](double v) { return log2(v); });
    }
    double terms[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) terms[j] = __shfl_sync(0xffffffffu, t, j);
    // flux (:110-124)
    const double sx = warp_np_sum([X](int64_t k) { return npy::dadd(X[k], f64::kEps); }, K, lane);
    const double sxp = warp_np_sum([Xp](int64_t k) { return npy::dadd(Xp[k], f64::kEps); }, K, lane);
    const double flux = warp_np_sum([X, Xp, sx, sxp](int64_t k) {
        const double d = npy::dsub(npy::ddiv(X[k], sx), npy::ddiv(Xp[k], sxp));
        return npy::dmul(d, d);
    }, K, lane);
    // rolloff (:127-140): np.cumsum runs in sequence
    double roll = 0.0;
    if (lane == 0) {
        const double thr = npy::dmul(0.90, tot);
        double c = 0.0;
        for (int k = 0; k < K; ++k) {
            c = npy::dadd(c, npy::dmul(X[k], X[k]));
            if (npy::dadd(c, EPS) > thr) { roll = npy::ddiv(double(k), double(K)); break; }
        }
    }
    // mfcc (:236-254): the mel filters' dot products, log10, the DCT rows
    for (int i = lane; i < B200AA_N_MEL; i += 32) {
        const int s0 = p.mel_idx[i], cnt = p.mel_idx[40 + i], off = p.mel_idx[80 + i];
        double acc = 0.0;
        for (int j = 0; j < cnt; ++j) acc = npy::dadd(acc, npy::dmul(p.mel_w[off + j], X[s0 + j]));
        scr[i] = log10(npy::dadd(acc, EPS));
    }
    __syncwarp();
    if (lane < B200AA_N_MFCC) {
        double acc = 0.0;
        for (int n = 0; n < B200AA_N_MEL; ++n) acc = npy::dadd(acc, npy::dmul(p.dct[lane * B200AA_N_MEL + n], scr[n]));
        out[size_t(8 + lane) * p.t_stride] = acc;
    }
    __syncwarp();
    // chroma (:277-321) and its population std (:667)
    const double ch = f64_chroma(p, X, tot, lane);
    if (lane < 12) {
        scr[lane] = ch;
        out[size_t(21 + lane) * p.t_stride] = ch;
    }
    __syncwarp();
    if (lane == 0) {
        double m, sd;
        front::pool_window([scr](int64_t i) { return scr[i]; }, 12, m, sd);
        out[size_t(3) * p.t_stride] = npy::ddiv(cen, npy::ddiv(fs, 2.0));
        out[size_t(4) * p.t_stride] = npy::ddiv(spr, npy::ddiv(fs, 2.0));
        out[size_t(5) * p.t_stride] = f64::entropy_of(terms);
        out[size_t(6) * p.t_stride] = flux;
        out[size_t(7) * p.t_stride] = roll;
        out[size_t(33) * p.t_stride] = sd;
    }
    __syncwarp();
}

template <int MODE, bool BIG>
__global__ void __launch_bounds__(32) f64_frames_kernel(const F64Params p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x, w = p.window, s = p.step, K = p.K;
    unsigned char *const base = BIG ? p.scratch + size_t(blockIdx.x) * p.warp_bytes : smem_raw;
    double2 *const A = reinterpret_cast<double2 *>(base);
    double2 *const B = A + f64_buf_len(w);
    double *Xc = reinterpret_cast<double *>(B + f64_buf_len(w)), *Xq = Xc + K;

    for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const int64_t b = item / p.segs_per_clip, seg = item - b * p.segs_per_clip;
        const int64_t len = clip_len(p.len, b, p.n_samples);
        int64_t n_rows, n_full, n_it;
        if (MODE == kModeFeatures) {
            n_rows = n_full = n_it = rows::frames(len, w, s);
        } else {
            const rows::Rows r = MODE == kModeSpectrogram ? rows::spectrogram(len, w, s) : rows::chromagram(len, w, s);
            // a uniform batch writes every row of the launch; a ragged one the clip's own rows, none when refused
            n_rows = p.len ? (r.refused ? 0 : r.R) : p.rows_launch;
            n_full = r.n_full;
            n_it = r.n_it;
        }
        const int64_t t0 = seg * p.seg_len;
        if (t0 >= n_rows) continue;
        const int64_t t1 = min(t0 + p.seg_len, n_rows);
        const b200aa_clip_norm_f64 nm = p.norm[b];
        const void *clip = static_cast<const char *>(p.sig) + size_t(b) * p.clip_stride * sample_bytes(p.dtype);
        __syncwarp();

        if (MODE == kModeFeatures) {
            double *const col = p.out + size_t(b) * p.n_out * p.t_stride;
            // the frame before the segment gives the flux its previous spectrum; frame 0 is its own previous frame
            for (int64_t t = t0 > 0 ? t0 - 1 : 0; t < t1; ++t) {
                double time[3];
                double2 *freeb = f64_spectrum(p, clip, nm, t * s, w, A, B, Xc, t >= t0 ? time : nullptr, lane);
                if (t >= t0) {
                    double *o = col + t;
                    if (lane == 0) {
                        o[0] = time[0];
                        o[p.t_stride] = time[1];
                        o[2 * p.t_stride] = time[2];
                    }
                    f64_spectral(p, Xc, t == 0 ? Xc : Xq, reinterpret_cast<double *>(freeb), o, lane);
                }
                double *t_ = Xc; Xc = Xq; Xq = t_;          // this frame's spectrum is the next one's previous
                __syncwarp();
            }
            continue;
        }
        for (int64_t i = t0; i < t1; ++i) {
            const int64_t start = rows::frame_start(w, s, i);
            const bool full = i < n_full, filled = i < n_it;
            if (filled) f64_spectrum(p, clip, nm, start, full ? w : int(len - start), A, B, Xc, nullptr, lane);
            if (MODE == kModeSpectrogram) {
                double *o = p.out + (size_t(b) * p.rows_launch + i) * K;
                for (int k = lane; k < K; k += 32) o[k] = filled ? Xc[k] : 0.0;
            } else {
                double ch = 0.0;
                if (filled) ch = f64_chroma(p, Xc, sum_sq(Xc, K, lane), lane);
                if (lane < 12) p.out[(size_t(b) * p.rows_launch + i) * 12 + lane] = ch;
            }
            __syncwarp();
        }
    }
}

// the delta rows (:672-678): row 34 + f of frame t is fv_t - fv_{t-1}, 0 at t = 0; one thread per (clip, row, frame)
__global__ void __launch_bounds__(256) f64_deltas_kernel(double *out, int64_t n_clips, int64_t T, int64_t t_stride,
                                                         const int64_t *len, int64_t n_samples, int w, int s)
{
    const int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (e >= n_clips * B200AA_N_BASE * T) return;
    const int64_t t = e % T, bf = e / T;
    const int64_t b = bf / B200AA_N_BASE, f = bf - b * B200AA_N_BASE;
    if (len && t >= rows::frames(clip_len(len, b, n_samples), w, s)) return;
    const double *row = out + (size_t(b) * 2 * B200AA_N_BASE + f) * t_stride;
    out[(size_t(b) * 2 * B200AA_N_BASE + B200AA_N_BASE + f) * t_stride + t] = t == 0 ? 0.0 : npy::dsub(row[t], row[t - 1]);
}

static void fill_f64(F64Params &q, const PlanF64 &pl, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                     int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm_f64 *d_norm, double *d_out)
{
    const F64Tables &t = *pl.tables;
    std::memset(&q, 0, sizeof q);
    q.sig = d_sig; q.len = d_len; q.norm = d_norm; q.out = d_out;
    q.tw = static_cast<const double2 *>(t.tw.get());
    q.mel_idx = static_cast<const int *>(t.mel_idx.get());
    q.mel_w = static_cast<const double *>(t.mel_w.get());
    q.dct = static_cast<const double *>(t.dct.get());
    q.chr_idx = static_cast<const int *>(t.chr_idx.get());
    q.chr_div = static_cast<const double *>(t.chr_div.get());
    q.n_clips = n_clips; q.n_samples = n_samples; q.clip_stride = clip_stride;
    q.dtype = dtype; q.fs = pl.fs; q.window = pl.window; q.step = pl.step; q.K = pl.K;
    q.nrad = int(t.radix.size());
    for (int i = 0; i < q.nrad; ++i) q.radix[i] = t.radix[i];
}

// one launch of f64_frames_kernel over rows [0, rows) of every clip; arrays past the per-CTA shared-memory maximum
// (windows above ~4700 samples: the 1 s windows of music_thumbnailing) go to stream-ordered global scratch
template <int MODE>
static int launch_frames(const PlanF64 &pl, F64Params &q, int64_t rows, cudaStream_t st)
{
    constexpr size_t kSmemCap = 226 * 1024;
    constexpr int64_t kSeg = 16;                // frames per work item: the flux's extra frame costs 1 / 16
    q.seg_len = std::max<int64_t>(1, std::min<int64_t>(kSeg, rows));
    q.segs_per_clip = std::max<int64_t>(1, (rows + q.seg_len - 1) / q.seg_len);
    q.n_items = q.segs_per_clip * q.n_clips;
    if (q.n_items == 0 || rows <= 0) return B200AA_OK;
    q.warp_bytes = f64_warp_bytes(q.window, q.K);
    if (q.warp_bytes <= kSmemCap) {
        auto kern = f64_frames_kernel<MODE, false>;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kSmemCap)));
        int occ = 1;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 32, q.warp_bytes));
        const int64_t grid = std::min<int64_t>(q.n_items, int64_t(pl.sm_count) * std::max(occ, 1) * 4);
        kern<<<(unsigned)grid, 32, q.warp_bytes, st>>>(q);
        CK_LAUNCH("f64_frames_kernel");
        return B200AA_OK;
    }
    // one warp's arrays per CTA (1.76 MB at a 1 s window at 44.1 kHz): two CTAs per SM bound the scratch at ~465 MB
    const int64_t grid = std::min<int64_t>(q.n_items, int64_t(pl.sm_count) * 2);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(q.warp_bytes * size_t(grid));
    if (rc != B200AA_OK) return rc;
    q.scratch = static_cast<unsigned char *>(scratch.get());
    f64_frames_kernel<MODE, true><<<(unsigned)grid, 32, 0, st>>>(q);
    return scratch.done(launched("f64_frames_kernel (large window)"));
}

static bool f64_dtype_ok(int dtype)
{
    return dtype == B200AA_DTYPE_I16 || dtype == B200AA_DTYPE_F32 || dtype == B200AA_DTYPE_F64;
}

extern "C" int b200aa_st_features_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                      int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                      const b200aa_clip_norm_f64 *d_norm, int deltas, double *d_out, int64_t t_stride,
                                      void *stream)
{
    NvtxRange nvtx_("b200aa_st_features_f64");
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || !f64_dtype_ok(dtype) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    PlanF64 pl;
    int rc = plan_f64(plan, pl);
    if (rc != B200AA_OK) return rc;
    // error order of the reference: mel bank (before the loop), no frames (:684), chroma (frame 0)
    if (pl.tables_status == B200AA_ERR_MEL_RANGE) return B200AA_ERR_MEL_RANGE;
    const int64_t T = rows::frames(n_samples, pl.window, pl.step);
    if (T == 0) return B200AA_ERR_TOO_SHORT;
    if (pl.tables_status != B200AA_OK) return pl.tables_status;
    if ((rc = plan_f64_device(plan)) != B200AA_OK) return rc;       // where b200aa_st_features checks it
    if (t_stride < T) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = plan_f64_tables(plan, pl, st, "b200aa_st_features_f64")) != B200AA_OK) return rc;
    F64Params q;
    fill_f64(q, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    q.t_stride = t_stride;
    q.n_out = deltas ? 2 * B200AA_N_BASE : B200AA_N_BASE;
    if ((rc = launch_frames<kModeFeatures>(pl, q, T, st)) != B200AA_OK || !deltas) return rc;
    const int64_t n = n_clips * B200AA_N_BASE * T;
    f64_deltas_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_out, n_clips, T, t_stride, d_len, n_samples,
                                                                   pl.window, pl.step);
    CK_LAUNCH("f64_deltas_kernel");
    return B200AA_OK;
}

// b200aa_spectrogram_f64 / _ragged_f64 (d_len set); argument checks and refusals as b200aa_spectrogram's
static int spectrogram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                           int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm_f64 *d_norm, double *d_out,
                           void *stream)
{
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || !f64_dtype_ok(dtype) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    PlanF64 pl;
    int rc = plan_f64(plan, pl);
    if (rc != B200AA_OK) return rc;
    const rows::Rows r = rows::spectrogram(n_samples, pl.window, pl.step);
    if (r.refused) return B200AA_ERR_TOO_SHORT;
    if (n_clips == 0) return B200AA_OK;
    const char *entry = d_len ? "b200aa_spectrogram_ragged_f64" : "b200aa_spectrogram_f64";
    if ((rc = plan_f64_tables(plan, pl, static_cast<cudaStream_t>(stream), entry)) != B200AA_OK) return rc;
    F64Params q;
    fill_f64(q, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    q.rows_launch = r.R;
    return launch_frames<kModeSpectrogram>(pl, q, r.R, static_cast<cudaStream_t>(stream));
}

extern "C" int b200aa_spectrogram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                      int64_t n_samples, int64_t clip_stride, const b200aa_clip_norm_f64 *d_norm,
                                      double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_spectrogram_f64");
    return spectrogram_f64(plan, d_sig, dtype, n_clips, n_samples, clip_stride, nullptr, d_norm, d_out, stream);
}

extern "C" int b200aa_spectrogram_ragged_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                             int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                             const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_spectrogram_ragged_f64");
    if (!d_len) return B200AA_ERR_INVALID;
    return spectrogram_f64(plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream);
}

// b200aa_chromagram_f64 / _ragged_f64 (d_len set); argument checks and refusals as b200aa_chromagram's.  Clipped frames
// are transformed in the same launch as the full ones.
static int chromagram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                          int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm_f64 *d_norm, double *d_out,
                          void *stream)
{
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || !f64_dtype_ok(dtype) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    PlanF64 pl;
    int rc = plan_f64(plan, pl);
    if (rc != B200AA_OK) return rc;
    const int w = pl.window, s = pl.step;
    const rows::Rows r = rows::chromagram(n_samples, w, s);
    if (r.R <= 0 || (!d_len && n_samples - s - w < 0)) return B200AA_ERR_TOO_SHORT;
    if (pl.tables_status == B200AA_ERR_CHROMA) return B200AA_ERR_CHROMA;
    if (n_clips == 0) return B200AA_OK;
    if (!d_len && r.refused) return B200AA_ERR_INVALID;
    const char *entry = d_len ? "b200aa_chromagram_ragged_f64" : "b200aa_chromagram_f64";
    if ((rc = plan_f64_tables(plan, pl, static_cast<cudaStream_t>(stream), entry)) != B200AA_OK) return rc;
    F64Params q;
    fill_f64(q, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    q.rows_launch = r.R;
    return launch_frames<kModeChromagram>(pl, q, r.R, static_cast<cudaStream_t>(stream));
}

extern "C" int b200aa_chromagram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                     int64_t n_samples, int64_t clip_stride, const b200aa_clip_norm_f64 *d_norm,
                                     double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_chromagram_f64");
    return chromagram_f64(plan, d_sig, dtype, n_clips, n_samples, clip_stride, nullptr, d_norm, d_out, stream);
}

extern "C" int b200aa_chromagram_ragged_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                            int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                            const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_chromagram_ragged_f64");
    if (!d_len) return B200AA_ERR_INVALID;
    return chromagram_f64(plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream);
}

// ------------------------------------------------------------------------------------------------
// kernel 12c: mid-term pooling and the long-term mean of float64 rows, bit for bit NumPy
// ------------------------------------------------------------------------------------------------
// one thread per (clip, row, window); frames (nullable): clip b has T_b = clamp(frames[b], 0, t_stride) frames and writes
// only its own windows
__global__ void __launch_bounds__(256) f64_mid_pool_kernel(const double *st, int64_t n_clips, int F, int64_t T,
                                                           int64_t t_stride, const int64_t *frames, int ratio, int stepr,
                                                           int64_t M, double *mid)
{
    const int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (e >= n_clips * F * M) return;
    const int64_t j = e % M, bf = e / M;
    const int64_t b = bf / F;
    const int f = int(bf - b * F);
    if (frames) {
        T = min(max(frames[b], int64_t(0)), t_stride);
        if (j >= rows::windows_of(T, stepr)) return;
    }
    const double *row = st + (size_t(b) * F + f) * t_stride;
    double mean, sd;
    f64::mid_window([row](int64_t c) { return row[c]; }, T, j, ratio, stepr, mean, sd);
    mid[(size_t(b) * 2 * F + f) * M + j] = mean;
    mid[(size_t(b) * 2 * F + F + f) * M + j] = sd;
}

static int mid_pool_f64_launch(const double *d_st, int64_t n_clips, int n_feats, int64_t T, int64_t t_stride,
                               const int64_t *d_frames, int ratio, int step_ratio, double *d_mid, void *stream)
{
    const int64_t M = rows::windows_of(T, step_ratio);
    const int64_t n = n_clips * n_feats * M;
    if (n == 0) return B200AA_OK;
    f64_mid_pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        d_st, n_clips, n_feats, T, t_stride, d_frames, ratio, step_ratio, M, d_mid);
    CK_LAUNCH("f64_mid_pool_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_mid_pool_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                                   int ratio, int step_ratio, double *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool_f64");
    if (!d_st || !d_mid || n_clips < 0 || n_feats < 1 || n_frames < 1 || step_ratio < 1 || t_stride < n_frames)
        return B200AA_ERR_INVALID;
    return mid_pool_f64_launch(d_st, n_clips, n_feats, n_frames, t_stride, nullptr, ratio, step_ratio, d_mid, stream);
}

extern "C" int b200aa_mid_pool_ragged_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t t_stride,
                                          const int64_t *d_frames, int ratio, int step_ratio, double *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool_ragged_f64");
    if (!d_st || !d_frames || !d_mid || n_clips < 0 || n_feats < 1 || step_ratio < 1 || t_stride < 0)
        return B200AA_ERR_INVALID;
    return mid_pool_f64_launch(d_st, n_clips, n_feats, t_stride, t_stride, d_frames, ratio, step_ratio, d_mid, stream);
}

// one thread per (clip, row): the mean of its first M_b = clamp(windows[b], 0, M) columns (all M without windows)
__global__ void __launch_bounds__(256) f64_long_term_mean_kernel(const double *mid, int64_t all_rows, int n_rows, int64_t M,
                                                                 const int64_t *windows, double *out)
{
    const int64_t r = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (r >= all_rows) return;
    const int64_t Mb = windows ? min(max(windows[r / n_rows], int64_t(0)), M) : M;
    const double *row = mid + size_t(r) * M;
    out[r] = f64::long_term_mean([row](int64_t c) { return row[c]; }, Mb);
}

static int long_term_mean_f64_launch(const double *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                     const int64_t *d_windows, double *d_out, void *stream)
{
    const int64_t rows_ = n_clips * n_rows;
    if (rows_ == 0) return B200AA_OK;
    f64_long_term_mean_kernel<<<(unsigned)((rows_ + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        d_mid, rows_, n_rows, m_stride, d_windows, d_out);
    CK_LAUNCH("f64_long_term_mean_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_long_term_mean_f64(const double *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, double *d_out,
                                         void *stream)
{
    NvtxRange nvtx_("b200aa_long_term_mean_f64");
    if (!d_mid || !d_out || n_clips < 0 || n_rows < 1 || n_windows < 1) return B200AA_ERR_INVALID;
    return long_term_mean_f64_launch(d_mid, n_clips, n_rows, n_windows, nullptr, d_out, stream);
}

extern "C" int b200aa_long_term_mean_ragged_f64(const double *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                                const int64_t *d_windows, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_long_term_mean_ragged_f64");
    if (!d_mid || !d_windows || !d_out || n_clips < 0 || n_rows < 1 || m_stride < 0) return B200AA_ERR_INVALID;
    return long_term_mean_f64_launch(d_mid, n_clips, n_rows, m_stride, d_windows, d_out, stream);
}
