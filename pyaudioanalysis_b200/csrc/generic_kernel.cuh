// Generic short-term kernel: any window length.  Mixed-radix Stockham transform in shared
// memory (one output element per thread per pass, arbitrary prime radices), then one warp per
// frame for the features.  This is the correctness baseline for every (fs, window, step); the
// register-tiled kernels in fast_kernel.cuh take over for the window lengths they specialise.
#pragma once
#include "common.cuh"
#include "dft_codelets.cuh"

namespace b200aa {

// bytes of the per-CTA arrays that scale with the window: transform ping-pong buffers + magnitude rows (+ previous frame)
inline size_t generic_big_bytes(int G, int Nc, int Kp)
{
    return (size_t(G) * Nc * sizeof(float2) * 2 + size_t(G + 1) * Kp * sizeof(float) + 15) & ~size_t(15);
}
// shared-memory bytes of the generic kernel for G frames per group (big = false: the window-sized arrays live in global memory)
inline size_t generic_smem_bytes(int G, int Nc, int Kp, int blob_words, bool big_in_smem = true)
{
    size_t b = big_in_smem ? generic_big_bytes(G, Nc, Kp) : 0;
    b += size_t(G + 1) * kFvStride * sizeof(float);          // feature rows (+ previous frame)
    b += size_t(kWarps) * B200AA_N_MEL * sizeof(float);      // mel scratch
    b += size_t(G + 1) * sizeof(float);                      // row sums
    b += size_t(kWarps) * 64 * sizeof(float) + 32 * sizeof(int4) + 16;   // time-domain parts + lane constants
    b += size_t(blob_words) * sizeof(int);
    return (b + 15) & ~size_t(15);
}
// frames per CTA group of the generic kernel: 8 while the arrays fit 100 KB (two CTAs per SM), else the largest of
// 4, 2, 1 that fits 226 KB (227 KB is the per-CTA opt-in maximum); 0 = one frame does not fit shared memory and the
// window-sized arrays go to global scratch
inline int generic_group(int Nc, int Kp, int blob_words)
{
    for (int G = 8; G >= 1; G >>= 1)
        if (generic_smem_bytes(G, Nc, Kp, blob_words) <= (G == 8 ? 100u * 1024u : 226u * 1024u)) return G;
    return 0;
}

// One Stockham pass of radix R with one BUTTERFLY per thread (R = 2, 3, 4, 5, 7: register codelets of
// dft_codelets.cuh); other radices use the one-output-per-thread form inside the kernel.
template <int R>
__device__ __forceinline__ void stockham_pass_bfly(const float2 *src, float2 *dst, int ng, int Nc, int Ns,
                                                   const float2 *__restrict__ tw, int tid)
{
    const int nb = Nc / R, tstep = Nc / (Ns * R);
    for (int e = tid; e < ng * nb; e += kThreads) {
        const int f = e / nb, j = e - f * nb;
        const int k = j % Ns;
        const float2 *in = src + size_t(f) * Nc + j;
        float2 v[R];
        v[0] = in[0];
        int idx = 0;
#pragma unroll
        for (int r = 1; r < R; ++r) {
            idx += k * tstep;                      // (k * r * tstep) < Nc because k < Ns and r < R
            v[r] = cmul(in[r * nb], __ldg(tw + idx));
        }
        dft_small<R>(v);
        float2 *out = dst + size_t(f) * Nc + (j - k) * R + k;
#pragma unroll
        for (int q = 0; q < R; ++q) out[q * Ns] = v[q];
    }
}

// BIG: windows whose transform does not fit shared memory (e.g. the 1 s windows of music_thumbnailing at 44.1 kHz,
// audioSegmentation.py:1137-1139): same code, the window-sized arrays of the CTA sit in global memory (L2 resident),
// __syncthreads() orders the passes as before.
// RAGGED (row modes only): every clip takes its own row counts from p.len (ragged_rows); a template flag so that the
// uniform launches keep their code.
template <int MODE, bool BIG = false, bool RAGGED = false>
__global__ void __launch_bounds__(kThreads, 2) st_generic_kernel(const StParams p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int G = p.G, Nc = p.Nc, K = p.K, Kp = p.Kp, w = p.window;
    unsigned char *const big = BIG ? p.scratch + size_t(blockIdx.x) * p.scratch_stride : smem_raw;
    float2 *bufA = reinterpret_cast<float2 *>(big);
    float2 *bufB = bufA + size_t(G) * Nc;
    float *Xrows = reinterpret_cast<float *>(bufB + size_t(G) * Nc);    // row 0 = previous frame
    float *fvrows = BIG ? reinterpret_cast<float *>(smem_raw) : Xrows + size_t(G + 1) * Kp;   // row 0 = previous frame
    float *mscr = fvrows + size_t(G + 1) * kFvStride;
    float *rowsum = mscr + kWarps * B200AA_N_MEL;
    float *tparts = rowsum + ((G + 1 + 3) & ~3);
    int4 *tlane = reinterpret_cast<int4 *>(tparts + kWarps * 64);
    int *blob_s = reinterpret_cast<int *>(tlane + 32);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < p.bl.words; i += kThreads) blob_s[i] = p.blob[i];
    if (tid < 32) tlane[tid] = time_lane_init(w, tid);
    __syncthreads();
    const SmallTables tb = bind_tables(blob_s, p.bl);

    for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const int64_t b = item / p.segs_per_clip, seg = item % p.segs_per_clip;
        const int64_t len = p.len ? p.len[b] : p.n_samples;
        int64_t n_rows, n_valid;
        if (MODE == kModeFeatures) {
            n_rows = n_valid = len < w ? 0 : (len - w) / p.step + 1;     // loop guard :608
        } else {
            n_rows = p.rows_launch;
            n_valid = p.rows_valid;
            if constexpr (RAGGED) ragged_rows<MODE>(p, b, n_rows, n_valid);
        }
        const int64_t t0 = seg * p.seg_len;
        if (t0 >= n_rows) continue;
        const int64_t t1 = min(t0 + p.seg_len, n_rows);
        const b200aa_clip_norm nm = p.norm[b];
        const char *clip = reinterpret_cast<const char *>(p.sig) +
                           size_t(b) * p.clip_stride * (p.dtype == B200AA_DTYPE_I16 ? 2 : 4);
        const SampleReader rd{clip, p.dtype, nm.m};
        const int halo = (MODE == kModeFeatures) ? int(t0 < 2 ? t0 : 2) : 0;

        for (int64_t g0 = t0 - halo; g0 < t1; g0 += G) {
            const int ng = int((t1 - g0) < G ? (t1 - g0) : G);
            // ---- load: z[n] = (x[2n]-x0) + i (x[2n+1]-x0)   (or real only for odd windows)
            // Subtracting the frame's first sample makes constant frames transform to exact zeros,
            // as they (up to 1e-17) do in the float64 reference.
            for (int e = tid; e < ng * Nc; e += kThreads) {
                const int f = e / Nc, n = e - f * Nc;
                const int64_t fr = g0 + f;
                float2 z = make_float2(0.f, 0.f);
                if (fr < n_valid) {
                    const int64_t s0 = frame_first<MODE>(w, p.step, fr);
                    const float d0 = rd(s0);
                    if (p.packed) z = make_float2(rd(s0 + 2 * n) - d0, rd(s0 + 2 * n + 1) - d0);
                    else z = make_float2(rd(s0 + n) - d0, 0.f);
                }
                bufA[e] = z;
            }
            __syncthreads();
            if (MODE == kModeFeatures) {
                // time-domain rows from the staged samples (bufA holds x - x[frame start]; one warp per frame).
                // fvrows rows of this step are free: the previous step's store loop finished before its last barrier.
                for (int f = warp; f < ng; f += kWarps) {
                    const float2 *zf = bufA + size_t(f) * Nc;
                    const float d0 = rd(frame_first<MODE>(w, p.step, g0 + f));
                    float *fv = fvrows + size_t(f + 1) * kFvStride;
                    if (p.packed)
                        time_features_chunked([&](int n) { const float2 q = zf[n >> 1]; return ((n & 1) ? q.y : q.x) + d0; }, w, nm,
                                              tlane[lane], tparts + warp * 64, fv, lane);
                    else
                        time_features_chunked([&](int n) { return zf[n].x + d0; }, w, nm, tlane[lane], tparts + warp * 64, fv, lane);
                }
                // no barrier needed before the passes: they only read bufA as well
            }
            // ---- Stockham passes
            float2 *src = bufA, *dst = bufB;
            int Ns = 1;
            for (int ps = 0; ps < p.nrad; ++ps) {
                const int R = p.radix[ps];
                const int NsR = Ns * R, stride = Nc / R, tstep = Nc / NsR;
                if (R == 4) stockham_pass_bfly<4>(src, dst, ng, Nc, Ns, p.tw, tid);
                else if (R == 2) stockham_pass_bfly<2>(src, dst, ng, Nc, Ns, p.tw, tid);
                else if (R == 3) stockham_pass_bfly<3>(src, dst, ng, Nc, Ns, p.tw, tid);
                else if (R == 5) stockham_pass_bfly<5>(src, dst, ng, Nc, Ns, p.tw, tid);
                else if (R == 7) stockham_pass_bfly<7>(src, dst, ng, Nc, Ns, p.tw, tid);
                else
                for (int e = tid; e < ng * Nc; e += kThreads) {
                    const int f = e / Nc, o = e - f * Nc;
                    const int hi_ = o / NsR, rem = o - hi_ * NsR;
                    const int q = rem / Ns, k = rem - q * Ns;
                    const int j = hi_ * Ns + k;
                    int ph = (k * tstep + q * stride) % Nc;   // phase step per input
                    int idx = 0;
                    const float2 *in = src + size_t(f) * Nc + j;
                    // fp64 accumulation: a float sum of R terms errs by ~sqrt(R) u of its terms' size, which for large
                    // primes (and for the DC bin, whose partial sums of x - x0 grow with the offset of x0) exceeds the
                    // log2(N) u of the rest of the transform; products of floats are exact in fp64
                    double ax = 0.0, ay = 0.0;
                    for (int r = 0; r < R; ++r) {
                        const float2 t = __ldg(p.tw + idx);
                        const float2 v = in[r * stride];
                        ax = fma(double(v.x), double(t.x), fma(-double(v.y), double(t.y), ax));
                        ay = fma(double(v.x), double(t.y), fma(double(v.y), double(t.x), ay));
                        idx += ph;
                        if (idx >= Nc) idx -= Nc;
                    }
                    dst[e] = make_float2(float(ax), float(ay));
                }
                __syncthreads();
                float2 *t_ = src; src = dst; dst = t_;
                Ns = NsR;
            }
            // ---- magnitudes |X[k]| / K, k < K  (ShortTermFeatures.py:617-621).  Not unrolled: unrolled (and, in the BIG
            // form, unswitched on p.packed) the loop costs 250-300 instructions more per kernel and more registers.
#pragma unroll 1
            for (int e = tid; e < ng * K; e += kThreads) {
                const int f = e / K, k = e - f * K;
                const int64_t fr = g0 + f;
                float mag = 0.f;
                if (fr < n_valid) {
                    const float2 *Z = src + size_t(f) * Nc;
                    const float sc = nm.a / float(K);
                    float2 Xc;
                    if (p.packed) {
                        // k < K = Nc: X[k] from the pair (Z[k], Z[Nc-k]) of the half-length transform
                        const float2 zk = Z[k];
                        const float2 zm = Z[k == 0 ? 0 : Nc - k];
                        const float2 ev = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
                        const float2 od = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));
                        const float2 wk = __ldg(p.tw_post + k);
                        const float2 t = cmul(od, wk);
                        Xc = make_float2(ev.x + t.x, ev.y + t.y);
                    } else {
                        Xc = Z[k];
                    }
                    if (k == 0) {
                        // DC of y = a*(d - d0) + (a*d0 + bp):  a*sum(d-d0) + w*(a*d0+bp)
                        const float d0 = rd(frame_first<MODE>(w, p.step, fr));
                        mag = fabsf(fmaf(nm.a, Xc.x, float(w) * fmaf(nm.a, d0, nm.bp))) / float(K);
                    } else {
                        const float re = Xc.x * sc, im = Xc.y * sc;
                        mag = sqrtf(fmaf(re, re, im * im));
                    }
                }
                Xrows[size_t(f + 1) * Kp + k] = mag;
            }
            __syncthreads();

            if (MODE == kModeSpectrogram) {
                for (int e = tid; e < ng * K; e += kThreads) {
                    const int f = e / K, k = e - f * K;
                    p.out[(size_t(b) * p.rows_launch + (g0 + f)) * K + k] = Xrows[size_t(f + 1) * Kp + k];
                }
                __syncthreads();
                continue;
            }
            if (MODE == kModeChromagram) {
                for (int f = warp; f < ng; f += kWarps) {
                    const float *X = Xrows + size_t(f + 1) * Kp;
                    float sxx = 0.f;
                    for (int k = lane; k < K; k += 32) sxx = fmaf(X[k], X[k], sxx);
                    sxx = warp_sum(sxx);
                    const float ch = (g0 + f < n_valid) ? chroma_lane(X, sxx, tb, lane) : 0.f;
                    if (lane < 12) p.out[(size_t(b) * p.rows_launch + (g0 + f)) * 12 + lane] = ch;
                }
                __syncthreads();
                continue;
            }

            // ---- features: one warp per frame
            for (int f = warp; f < ng; f += kWarps) {
                const int64_t fr = g0 + f;
                const float *X = Xrows + size_t(f + 1) * Kp;
                // previous spectrum: row f (row 0 carries the last frame of the previous group);
                // the very first frame of a clip -- and a halo frame without history -- uses itself
                const bool has_prev = (fr > 0) && !(f == 0 && g0 == t0 - halo);
                float sxp;
                const float *Xp;
                float *fv = fvrows + size_t(f + 1) * kFvStride;
                if (has_prev && f > 0) {
                    // row sum of the neighbour is produced by another warp in this same phase:
                    // recompute it here instead of synchronising
                    Xp = Xrows + size_t(f) * Kp;
                    float s = 0.f;
                    for (int k = lane; k < K; k += 32) s += Xp[k];
                    sxp = warp_sum(s);
                } else if (has_prev) {
                    Xp = Xrows;
                    sxp = rowsum[0];
                } else {
                    Xp = X;
                    float s = 0.f;
                    for (int k = lane; k < K; k += 32) s += X[k];
                    sxp = warp_sum(s);
                }
                spectral_features(X, Xp, sxp, K, tb, mscr + warp * B200AA_N_MEL, fv, lane, rowsum + f + 1);
            }
            __syncthreads();
            // ---- store [n_out x ng] tile: consecutive threads -> consecutive frames
            for (int e = tid; e < p.n_out * ng; e += kThreads) {
                const int f = e / ng, c = e - f * ng;
                const int64_t fr = g0 + c;
                if (fr < t0) continue;
                float v;
                if (f < B200AA_N_BASE) v = fvrows[size_t(c + 1) * kFvStride + f];
                else {
                    const int fb = f - B200AA_N_BASE;
                    v = fr == 0 ? 0.f : fvrows[size_t(c + 1) * kFvStride + fb] - fvrows[size_t(c) * kFvStride + fb];
                }
                p.out[(size_t(b) * p.n_out + f) * p.t_stride + fr] = v;
            }
            __syncthreads();
            // ---- carry the last frame of the group into row 0
            for (int k = tid; k < K; k += kThreads) Xrows[k] = Xrows[size_t(ng) * Kp + k];
            if (tid < kFvStride) fvrows[tid] = fvrows[size_t(ng) * kFvStride + tid];
            if (tid == 0) rowsum[0] = rowsum[ng];
            __syncthreads();
        }
    }
}

// bytes of the clipped-frame kernel's per-CTA arrays: |X| row [K] (16-byte padded), twiddles [w] double2, samples [w] double
inline size_t clipped_bytes(int w, int K)
{
    return ((size_t(K) * sizeof(float) + 15) & ~size_t(15)) + size_t(w) * (sizeof(double2) + sizeof(double));
}

// Chromagram rows of the frames clipped at the end of a clip (ShortTermFeatures.py:349-355): row i >= n_full of clip b
// transforms the n = len - (w + i*s) samples left, K <= n < w (rows::chromagram).  Work item = (clip b, candidate c <
// per_clip): the row is n_full + c, and an item without such a row does nothing, so one launch serves every clip and
// every clipped length whether the lengths are known on the host or only on the device (p.len).
// Direct DFT of length n: z[j] = x[j] - x[0] in fp64, the phase index j*k mod n advances exactly in integers over a
// table of the n twiddles the CTA builds for this n, fp64 accumulation.  Then |X|[0:K] / K of y = a*(x - m) + bp (the
// DC bin adds n*(a*(x[0] - m) + bp)) rounded to float, and the chroma row with the plan's taps / sum(X^2) as in
// st_generic_kernel's chromagram mode.
// BIG: windows whose arrays do not fit shared memory keep them in global scratch (p.scratch, p.scratch_stride per CTA).
template <bool BIG>
__global__ void __launch_bounds__(kThreads, 2) clipped_chroma_kernel(const StParams p, int64_t per_clip)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int w = p.window, s = p.step, K = p.K;
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned char *const base = BIG ? p.scratch + size_t(blockIdx.x) * p.scratch_stride : smem_raw;
    float *const X = reinterpret_cast<float *>(base);
    double2 *const tw = reinterpret_cast<double2 *>(base + ((size_t(K) * sizeof(float) + 15) & ~size_t(15)));
    double *const z = reinterpret_cast<double *>(tw + w);
    const SmallTables tb = bind_tables(p.blob, p.bl);           // chroma taps straight from global memory
    const bool is16 = p.dtype == B200AA_DTYPE_I16;

    for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const int64_t b = item / per_clip, c = item - b * per_clip;
        const int64_t len = p.len ? ragged_len(p, b) : p.n_samples;
        const rows::Rows r = rows::chromagram(len, w, s);
        const int64_t i = r.n_full + c;
        if (r.refused || i >= r.n_it) continue;                 // uniform across the CTA
        const int64_t start = rows::frame_start(w, s, i);
        const int n = int(len - start);
        const char *clip = reinterpret_cast<const char *>(p.sig) + size_t(b) * p.clip_stride * (is16 ? 2 : 4);
        auto x = [&](int64_t j) -> double {
            return is16 ? double(reinterpret_cast<const short *>(clip)[start + j]) : double(reinterpret_cast<const float *>(clip)[start + j]);
        };
        const double x0 = x(0);
        __syncthreads();                                        // the previous item is done with X, tw and z
        for (int j = tid; j < n; j += kThreads) {
            z[j] = x(j) - x0;                                   // exact: a difference of two int16 / float32 values
            double sn, cs;
            sincospi(2.0 * double(j) / double(n), &sn, &cs);
            tw[j] = make_double2(cs, -sn);
        }
        __syncthreads();
        const b200aa_clip_norm nm = p.norm[b];
        const double a = nm.a;
        for (int k = tid; k < K; k += kThreads) {
            double re = 0.0, im = 0.0;
            int ph = 0;                                         // j*k mod n; k < K <= n
            for (int j = 0; j < n; ++j) {
                const double2 t = tw[ph];
                re = fma(z[j], t.x, re);
                im = fma(z[j], t.y, im);
                ph += k;
                if (ph >= n) ph -= n;
            }
            const double mag = k == 0 ? fabs(a * re + double(n) * (a * (x0 - double(nm.m)) + double(nm.bp))) : a * sqrt(re * re + im * im);
            X[k] = float(mag / double(K));
        }
        __syncthreads();
        if (tid < 32) {
            float sxx = 0.f;
            for (int k = lane; k < K; k += 32) sxx = fmaf(X[k], X[k], sxx);
            sxx = warp_sum(sxx);
            const float ch = chroma_lane(X, sxx, tb, lane);
            if (lane < 12) p.out[(size_t(b) * p.rows_launch + i) * 12 + lane] = ch;
        }
    }
}

}  // namespace b200aa
