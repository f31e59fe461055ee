// Register-tiled short-term kernel for even windows N = 2*R1*R2 (20x20 -> 800 samples = 50 ms @ 16 kHz,
// 21x21 -> 882 = 20 ms @ 44.1 kHz, 20x10 -> 400, 20x12 -> 480, 20x15 -> 600, 16x10 -> 320, 20x16 -> 640).
//
// The real frame is packed into Nc = R1*R2 complex points z[n] = x[2n] + i x[2n+1] and transformed as an
// R1 x R2 two-pass FFT: every pass is one small FFT per thread held entirely in registers (prime-factor
// 4x5 / 3x7 / 2x5 / 3x4 / 3x5 butterflies without internal twiddles, 4x4 Cooley-Tukey for 16; all
// constants are immediates, butterflies on float2 (re, im) pairs), with one padded shared-memory
// transpose between the passes.  max(R1, R2) threads own a frame; 8 frames per CTA step.  Post-processing
// computes |X[k]| and |X[Nc-k]| from one (Z[k], Z[Nc-k]) pair, so only half of the second-pass outputs
// travel through shared memory.  Samples arrive by TMA (cp.async.bulk + mbarrier) one step ahead.
#pragma once
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>
#include "common.cuh"
#include "dft_codelets.cuh"
#include "sched.cuh"
#include "tables.inl"

namespace b200aa {

#ifndef B200AA_FAST_G
#define B200AA_FAST_G 8       // frames per CTA step (CTA = 32*G threads)
#endif
#ifndef B200AA_FAST_MINBLOCKS
#define B200AA_FAST_MINBLOCKS 3   // CTAs per SM the fast kernel is compiled for (register budget)
#endif
// threads per CTA: one warp per frame slot
__host__ __device__ constexpr int fast_threads(int g) { return 32 * g; }

// ---- cheap math: MUFU-based reciprocal / rsqrt / log2 (2 ulp); every feature entry stays within its per-entry bound
// at these documented errors (tests/parity.feature_bounds, error model in tests/test_feature_bounds_cpu.py)
__device__ __forceinline__ float fdiv(float a, float b) { return __fdividef(a, b); }
// rsqrtf() is the MUFU.RSQ approximation; __frsqrt_rn() is the correctly rounded (slow) one -- measured 12 % slower
#ifndef B200AA_NO_FTZ_MUFU
__device__ __forceinline__ float fsqrt_pos(float x)      // bare MUFU.RSQ (flush-to-zero form: no denormal fix-up code)
{
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaxf(x, 1e-36f)));
    return x * r;
}
__device__ __forceinline__ float flog2(float x)
{
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
#else
__device__ __forceinline__ float fsqrt_pos(float x) { return x * rsqrtf(fmaxf(x, 1e-36f)); }   // 0 -> 0
__device__ __forceinline__ float flog2(float x) { return __log2f(x); }
#endif

template <int K>
struct DenseShape {
    static constexpr int C = ((K + 31) / 32) | 1;   // bins per lane (odd => conflict-free chunk loads)
    static constexpr int Kp = 32 * C;               // row length incl. zero padding: no bounds checks
    static constexpr int Lb = K / 10;               // spectral-entropy block length (:94)
};

// ----------------------------------------------------------------------------------------------
// Half-warp variant of the dense pass: 16 lanes per frame (a warp handles two frames), every lane holds
// C2 = odd(ceil(K/32)) float2 pairs of consecutive bins, per-bin arithmetic on float2 pairs.  The
// fixed per-frame overhead (reductions, scalar math, stores) is paid once per two frames.
// ----------------------------------------------------------------------------------------------
template <int K>
struct HalfShape {
    static constexpr int C2 = ((K + 31) / 32) | 1;      // float2 per lane (odd => conflict-free 8-byte loads)
    static constexpr int CB = 2 * C2;                   // bins per lane
    static constexpr int Lb = K / 10;
    static_assert(16 * CB == DenseShape<K>::Kp, "same padded row length as the warp-per-frame layout");
    static_assert(CB < Lb && (Lb % 2) == 0, "one (even) entropy block boundary per lane at most");
};
// per-lane constants of the half-warp dense pass (here and in pair_kernel.cuh / solo_kernel.cuh; depend on the lane only,
// computed once per CTA), l = lane within the half-warp, 0..15:
// .x = bins of the lane's chunk that belong to the earlier entropy block, [.y, .z) = parts (2 per lane, in bin order) of block l
template <int K>
__device__ __forceinline__ int4 pair_lane_init(int l)
{
    constexpr int CB = 2 * (((K + 31) / 32) | 1), Lb = K / 10;
    const int k0 = l * CB;
    const int bnd = ((k0 + CB - 1) / Lb) * Lb;
    int4 d;
    d.x = bnd > k0 ? bnd - k0 : 0;
    int ps = 32, pe = 0;
#pragma unroll 1
    for (int q = 0; q < 16; ++q) {
        const int b0 = q * CB, bb = ((b0 + CB - 1) / Lb) * Lb, sp = bb > b0 ? bb - b0 : 0;
        if (sp > 0 && b0 >= l * Lb && b0 + sp <= (l + 1) * Lb) { ps = min(ps, 2 * q); pe = max(pe, 2 * q + 1); }
        if (b0 + sp >= l * Lb && b0 + CB <= (l + 1) * Lb) { ps = min(ps, 2 * q + 1); pe = max(pe, 2 * q + 2); }
    }
    if (l >= 10) { ps = 0; pe = 0; }
    d.y = ps; d.z = pe; d.w = 0;
    return d;
}
__device__ __forceinline__ float half_sum(float v)      // sum over the 16 lanes of a half-warp (both halves at once)
{
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <int K>
__device__ __forceinline__ float row_sum_h(const float *X, int l)
{
    constexpr int C2 = HalfShape<K>::C2;
    const float2 *X2 = reinterpret_cast<const float2 *>(X) + l * C2;
    float sx = 0.f;
#pragma unroll
    for (int j = 0; j < C2; ++j) { const float2 v = X2[j]; sx += v.x + v.y; }
    return half_sum(sx);
}

template <int K>
__device__ __forceinline__ void spectral_features_h(const float *X, const float *Xp, float sxp,
                                                    const int *dlp, float *parts, float *fv, int l, bool active, float *xsave)
{
    constexpr int C2 = HalfShape<K>::C2, CB = HalfShape<K>::CB;
    const int k0 = l * CB;
    const int4 dlv = *reinterpret_cast<const int4 *>(dlp);        // {split (bins), ps, pe, -}
    const float2 *X2 = reinterpret_cast<const float2 *>(X) + l * C2;
    const float2 *Xp2 = reinterpret_cast<const float2 *>(Xp) + l * C2;
    float2 x2[C2];
#pragma unroll
    for (int j = 0; j < C2; ++j) x2[j] = X2[j];
    if (xsave) {
        float2 *S2 = reinterpret_cast<float2 *>(xsave) + l * C2;
#pragma unroll
        for (int j = 0; j < C2; ++j) S2[j] = x2[j];
    }
    // ---- sums (same per-lane order as row_sum_h)
    float sx = 0.f, s1 = 0.f, sb = 0.f;
    float2 plo2 = make_float2(0.f, 0.f), phi2 = make_float2(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < C2; ++j) {
        const float t = x2[j].x + x2[j].y;
        sx += t;
        s1 = fmaf(float(2 * j + 1), t, s1);          // (2j+1) a + (2j+2) b = (2j+1)(a+b) + b
        sb += x2[j].y;
        const float2 sq = f2mul(x2[j], x2[j]);
        if (2 * j < dlv.x) plo2 = f2add(plo2, sq); else phi2 = f2add(phi2, sq);     // Lb even: boundaries between pairs
    }
    const float plo = plo2.x + plo2.y, phi = phi2.x + phi2.y, part = plo + phi;
    float sk = fmaf(float(k0), sx, s1 + sb);         // sum (k0 + i + 1) x_i
    parts[2 * l] = plo;
    parts[2 * l + 1] = phi;
    {   // two sums in 4 exchanges: lanes 0-7 of the half end up with sum(sx), lanes 8-15 with sum(sk)
        const bool up = l & 8;
        float keep = up ? sk : sx;
        const float give = up ? sx : sk;
        keep += __shfl_xor_sync(0xffffffffu, give, 8);
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) keep += __shfl_xor_sync(0xffffffffu, keep, o);
        sx = __shfl_sync(0xffffffffu, keep, 0, 16);
        sk = __shfl_sync(0xffffffffu, keep, 8, 16);
    }
    float incl = part;
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
        const float n = __shfl_up_sync(0xffffffffu, incl, o, 16);
        if (l >= o) incl += n;
    }
    const float sxx = __shfl_sync(0xffffffffu, incl, 15, 16);
    constexpr float invK = 1.f / float(K);
    const float cen = sx > 0.f ? fdiv(sk, sx) * invK : 0.f;
    // ---- spread, flux, rolloff count
    const float nx = fdiv(1.f, sx + float(K) * B200AA_EPS);
    const float np_ = fdiv(1.f, sxp + float(K) * B200AA_EPS);
    const float thr = 0.90f * sxx - B200AA_EPS;
    float2 d2 = make_float2(float(k0 + 1) * invK - cen, float(k0 + 2) * invK - cen);
    const float2 dstep = make_float2(2.f * invK, 2.f * invK);
    const float2 nx2 = make_float2(nx, nx), mnp2 = make_float2(-np_, -np_);
    float2 sp2 = make_float2(0.f, 0.f), fl2 = make_float2(0.f, 0.f);
    float run = incl - part, below = 0.f;
#pragma unroll
    for (int j = 0; j < C2; ++j) {
        sp2 = f2fma(f2mul(d2, d2), x2[j], sp2);
        d2 = f2add(d2, dstep);
        const float2 df = f2fma(x2[j], nx2, f2mul(Xp2[j], mnp2));
        fl2 = f2fma(df, df, fl2);
        // padding bins never count: at the last real bin the running sum equals sxx > thr (or everything is 0)
        run = fmaf(x2[j].x, x2[j].x, run);
        below += run > thr ? 0.f : 1.f;
        run = fmaf(x2[j].y, x2[j].y, run);
        below += run > thr ? 0.f : 1.f;
    }
    const float sp = sp2.x + sp2.y, fl = fl2.x + fl2.y;
    // ---- spectral entropy: lanes 0..9 of the half add up the parts of their block
    __syncwarp();
    float e = 0.f;
    constexpr int MAXP = 2 * (HalfShape<K>::Lb / CB + 2);
#pragma unroll
    for (int q = 0; q < MAXP; ++q) e += (dlv.y + q < dlv.z) ? parts[dlv.y + q] : 0.f;
    float ent = 0.f;
    if (l < 10) {
        const float sj = fdiv(e, sxx + B200AA_EPS);
        ent = -sj * flog2(sj + B200AA_EPS);
    }
    // four sums in 4 exchanges: lanes 0-3 spread, 4-7 flux, 8-11 rolloff count, 12-15 entropy
    float q4;
    {
        const bool up8 = l & 8, up4 = l & 4;
        float k0_ = up8 ? below : sp, k1_ = up8 ? ent : fl;
        const float g0_ = up8 ? sp : below, g1_ = up8 ? fl : ent;
        k0_ += __shfl_xor_sync(0xffffffffu, g0_, 8);
        k1_ += __shfl_xor_sync(0xffffffffu, g1_, 8);
        float kk = up4 ? k1_ : k0_;
        const float gg = up4 ? k0_ : k1_;
        kk += __shfl_xor_sync(0xffffffffu, gg, 4);
        kk += __shfl_xor_sync(0xffffffffu, kk, 2);
        kk += __shfl_xor_sync(0xffffffffu, kk, 1);
        q4 = kk;
    }
    if (active) {
        if (l == 0) {
            fv[3] = cen;
            fv[4] = sx > 0.f ? fsqrt_pos(fdiv(q4, sx)) : 0.f;
            fv[34] = sx;
            fv[35] = sxx;                            // sum X^2: the chroma rows are normalised by it later
        }
        if (l == 4) fv[6] = q4;
        if (l == 8) fv[7] = q4 >= float(K) ? 0.f : q4 * invK;
        if (l == 12) fv[5] = q4;
    }
    __syncwarp();
}

// time-domain rows of two frames per warp (half-warp each; lanes 0..9 of a half own the ten entropy blocks)
template <int N>
__device__ __forceinline__ void time_features_runs_h(const float *runE, const int *runF, float *fv, int l, bool active)
{
    constexpr int RPB = N / 80;
    float e = 0.f;
    int f = 0;
    if (l < 10) {
#pragma unroll
        for (int i = 0; i < RPB; ++i) {
            e += runE[l * RPB + i];
            const int w = runF[l * RPB + i];
            f += (w & 0xff) + (w >> 8);
        }
    }
    const float tot = half_sum(e);
    int ft = f;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) ft += __shfl_xor_sync(0xffffffffu, ft, o);
    ft -= runF[0] >> 8;
    const float sj = fdiv(e, tot + B200AA_EPS);
    float H = l < 10 ? -sj * flog2(sj + B200AA_EPS) : 0.f;
    H = half_sum(H);
    if (active && l == 0) {
        fv[0] = float(ft) * 0.5f / float(N - 1);
        fv[1] = tot / float(N);
        fv[2] = H;
    }
}

// ---- mel + raw chroma on the upper half of the CTA (threads NT/2 .. NT-1) while the lower half runs the dense
// pass: 16 threads per frame, every thread a group of <= 3 filters with balanced tap totals; then 12 threads per
// frame for the chroma tap sums
template <int G, int UT = 16 * G>
__device__ __forceinline__ void upper_mel_chroma(const float *Xrows, int Kp, int ng, const SmallTables &tb, const int *grp_tab,
                                                 float *ms, float *chr, int t0)
{
    // UT threads (t0 < UT) share the G * 16 (frame, filter group) slots and the G * 12 (frame, pitch class) slots
    static_assert((16 * G) % UT == 0, "whole rounds over the filter-group slots");
#pragma unroll
    for (int rd = 0; rd < (16 * G) / UT; ++rd) {
        const int t = t0 + rd * UT;
        const int f = t >> 4, sub = t & 15;
        if (f < ng) {
            const float *X = Xrows + size_t(f) * Kp;
#pragma unroll
            for (int h = 0; h < 3; ++h) {
                const int i = grp_tab[3 * sub + h];
                if (i >= 0) {
                    const int s0 = tb.mel_start[i], cnt = tb.mel_count[i], off = tb.mel_off[i];
                    float acc = 0.f;
#pragma unroll 4
                    for (int q = 0; q < cnt; ++q) acc = fmaf(X[s0 + q], tb.mel_w[off + q], acc);
                    ms[f * B200AA_N_MEL + i] = 0.30102999566398120f * flog2(acc + B200AA_EPS);   // log10
                }
            }
        }
    }
#pragma unroll
    for (int rd = 0; rd < (G * 12 + UT - 1) / UT; ++rd) {
        const int t = t0 + rd * UT;
        if (t >= G * 12) continue;
        const int f = t / 12, c = t - f * 12;
        if (f < ng) {
            const float *X = Xrows + size_t(f) * Kp;
            const int e0 = tb.chr_off[c], e1 = tb.chr_off[c + 1];
            float acc = 0.f;
            for (int e = e0; e < e1; ++e) {
                const float v = X[tb.chr_bin[e]];
                acc = fmaf(v * v, tb.chr_w[e], acc);
            }
            chr[f * 12 + c] = acc;
        }
    }
}

// chroma rows of two frames per warp: normalise the tap sums by sum X^2 (fv[35]) and add their population std
__device__ __forceinline__ void chroma_finalize_h(const float *chroma_raw, float *fv, int l, bool active)
{
    const float sxx = fv[35];
    const float ch = l < 12 ? fdiv(chroma_raw[l], sxx == 0.f ? B200AA_EPS : sxx) : 0.f;
    const float mean = half_sum(ch) * (1.f / 12.f);
    const float dv = l < 12 ? ch - mean : 0.f;
    const float var = half_sum(dv * dv) * (1.f / 12.f);
    if (active) {
        if (l < 12) fv[21 + l] = ch;
        if (l == 0) fv[33] = fsqrt_pos(var);
    }
}

// ---- DCT: threads 0..207 = (frame, cepstral row c, half h): folded DCT-II
//   y_c = sum_{n<20} D[c][n] * ((m_n - k) + (-1)^c (m_{39-n} - k)),  k = m_0 (any constant works for
//   c >= 1 because those rows are orthogonal to constants; row 0 adds it back): keeps the float32 sum
//   free of the large common offset of the log-mel values.
template <int G, int NT = 32 * G>
__device__ __forceinline__ void flat_dct(const float *ms, int ng, const SmallTables &tb, float *fvrows, int fbase, int tid0)
{
    static_assert(NT % 2 == 0, "the two halves of a row sit in neighbouring lanes");
#pragma unroll
    for (int base = 0; base < G * 26; base += NT) {       // every thread runs every round (the shuffle needs whole warps)
    const int tid = base + tid0;
    const int f = tid / 26, r = tid - f * 26;
    const int c = r >> 1, h = r & 1;
    float acc = 0.f;
    const bool act = tid < G * 26 && f < ng;
    if (act) {
        const float *m = ms + f * B200AA_N_MEL;
        const float kap = m[0];
        const float *row = tb.dct + c * 41;
        const float sgn = (c & 1) ? -1.f : 1.f;
#pragma unroll
        for (int j = 0; j < 10; ++j) {
            const int n = 10 * h + j;
            const float a = m[n] - kap, b = m[39 - n] - kap;
            acc = fmaf(row[n], fmaf(sgn, b, a), acc);
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (act && h == 0) {
        if (c == 0) acc = fmaf(6.324555320336759f, ms[f * B200AA_N_MEL], acc);    // sqrt(1/40) * 40 * k
        int r = fbase + 1 + f;
        if (r > G) r -= G + 1;
        fvrows[r * kFvStride + 8 + c] = acc;
    }
    }
}

// ----------------------------------------------------------------------------------------------
// staging fused with the time-domain partials.  One thread converts one run of 8 consecutive
// samples (one 16-byte load of int16), stores x - m to shared memory and emits for the run:
//   runE = sum y^2                      (y = a (x-m) + bp, energy / energy-entropy, :29-51)
//   runF = sign flips inside the run + (flip between the run's first sample and its predecessor) << 8
// Frames are whole numbers of runs (N % 80 == 0, step % 8 == 0), so zcr / energy / block energies of
// a frame are sums over its 100 runs and the 50 % overlap is computed once.
// ----------------------------------------------------------------------------------------------

__device__ __forceinline__ void stage_run(const void *clip, int dtype, bool vec_ok, int64_t n0, const b200aa_clip_norm &nm,
                                          float *dst, float *runE, int *runF)
{
    float d[8];
    if (dtype == B200AA_DTYPE_I16) {
        const short *x = reinterpret_cast<const short *>(clip) + n0;
        if (vec_ok) {
            const int4 q = __ldg(reinterpret_cast<const int4 *>(x));
            const int w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                d[2 * u] = float((short)(w4[u] & 0xffff)) - nm.m;
                d[2 * u + 1] = float(w4[u] >> 16) - nm.m;
            }
        } else {
#pragma unroll
            for (int u = 0; u < 8; ++u) d[u] = float(x[u]) - nm.m;
        }
    } else {
        const float *x = reinterpret_cast<const float *>(clip) + n0;
        if (vec_ok) {
            const float4 q0 = __ldg(reinterpret_cast<const float4 *>(x)), q1 = __ldg(reinterpret_cast<const float4 *>(x) + 1);
            d[0] = q0.x - nm.m; d[1] = q0.y - nm.m; d[2] = q0.z - nm.m; d[3] = q0.w - nm.m;
            d[4] = q1.x - nm.m; d[5] = q1.y - nm.m; d[6] = q1.z - nm.m; d[7] = q1.w - nm.m;
        } else {
#pragma unroll
            for (int u = 0; u < 8; ++u) d[u] = x[u] - nm.m;
        }
    }
    float e = 0.f, fl = 0.f, s[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const float y = fmaf(nm.a, d[u], nm.bp);
        e = fmaf(y, y, e);
        s[u] = sign_class(d[u], nm.lo, nm.hi);
        if (u > 0) fl += fabsf(s[u] - s[u - 1]);
    }
    float linkf = 0.f;
    if (n0 > 0) {
        const float dp = (dtype == B200AA_DTYPE_I16 ? float(reinterpret_cast<const short *>(clip)[n0 - 1])
                                                    : reinterpret_cast<const float *>(clip)[n0 - 1]) - nm.m;
        linkf = fabsf(s[0] - sign_class(dp, nm.lo, nm.hi));
    }
    const int link = int(linkf);
    const int fli = int(fl);
    *reinterpret_cast<float4 *>(dst) = make_float4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<float4 *>(dst + 4) = make_float4(d[4], d[5], d[6], d[7]);
    *runE = e;
    *runF = fli | (link << 8);
}

// ----------------------------------------------------------------------------------------------
// TMA (1-D bulk async copy) + mbarrier: the raw int16 samples of the NEXT CTA step are fetched from
// HBM into shared memory by the copy engine while this step's FFT / features run
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar)
{
    // order the CTA's earlier generic-proxy reads of the buffer before the async-proxy write
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
    unsigned done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
    } while (!done);
}

// stage_run() with the 8 int16 samples (and their predecessor) already in shared memory
__device__ __forceinline__ void stage_run_smem(const short *raw8, bool has_pred, const b200aa_clip_norm &nm, float *dst, float *runE,
                                               int *runF)
{
    const int4 q = *reinterpret_cast<const int4 *>(raw8);
    const int w4[4] = {q.x, q.y, q.z, q.w};
    float d[8];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        d[2 * u] = float((short)(w4[u] & 0xffff)) - nm.m;
        d[2 * u + 1] = float(w4[u] >> 16) - nm.m;
    }
    float e = 0.f, fl = 0.f, s[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const float y = fmaf(nm.a, d[u], nm.bp);
        e = fmaf(y, y, e);
        s[u] = sign_class(d[u], nm.lo, nm.hi);
        if (u > 0) fl += fabsf(s[u] - s[u - 1]);
    }
    float linkf = 0.f;
    if (has_pred) linkf = fabsf(s[0] - sign_class(float(raw8[-1]) - nm.m, nm.lo, nm.hi));
    *reinterpret_cast<float4 *>(dst) = make_float4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<float4 *>(dst + 4) = make_float4(d[4], d[5], d[6], d[7]);
    *runE = e;
    *runF = int(fl) | (int(linkf) << 8);
}

// ----------------------------------------------------------------------------------------------
// kernel
// ----------------------------------------------------------------------------------------------
struct FastTables {
    b200aa_host::DeviceMemory tw;      // float2 [R][R]   W_Nc^(k1*n2) stored [k1][n2]
    b200aa_host::DeviceMemory twp;     // float2 [Nc/2+1] W_N^k
    int R = 0;
};


// Nc = R1 * R2 complex points per frame: n = R2*n1 + n2, k = k1 + R1*k2.  Pass 1: R2 threads per frame, each an
// R1-point FFT over n1; pass 2 / post-processing: R1 threads per frame, each an R2-point FFT over n2.
template <int R1, int R2, int G>
struct FastShape {
    static constexpr int Nc = R1 * R2, N = 2 * Nc, K = Nc, Kp = DenseShape<Nc>::Kp;   // rows zero-padded to 32*C bins
    static constexpr int TPF = R1 > R2 ? R1 : R2;   // threads that own a frame during the transform
    static constexpr int ES = R2 | 1;            // padded row stride of the transpose buffer [R1][ES] (float2)
    static constexpr int H = R2 / 2;             // second-pass outputs k2 >= H are published for the partners
    static constexpr int ZS = Nc - R1 * H;       // published values per frame
    static constexpr int FftThreads = G * TPF;
    static_assert(TPF <= 32, "one frame's transform threads fit a warp-sized slot");
    static constexpr int NT = 32 * G;            // threads per CTA
};

// fixed-size part of the CTA's shared memory (compile-time offsets)
template <int R1, int R2, int G>
struct alignas(16) FastFixed {
    using S = FastShape<R1, R2, G>;
    float2 E[G * R1 * S::ES];              // transpose buffer [G][R][ES]; the |X| rows alias it
    float2 tw[R1 * R2];                   // W_Nc^(k1 n2)  [k1][n2]
    float2 twp[(S::Nc / 2 + 2) & ~1];     // W_N^k
    alignas(16) float Xprev[2 * S::Kp];   // |X| of the previous step's last frame (double-buffered)
    float fvrows[(G + 1) * kFvStride];    // ring of feature rows: 34 features + the row's sum(X) in slot 34
    float mscr[G * B200AA_N_MEL];         // log-mel energies
    float chr[G * 12];                    // raw chroma sums
    float parts[G * 64];                  // entropy parts per (dense) half-warp; the chunked time-domain pass needs 64 per warp
    alignas(16) int dlane[32 * 4];        // per-lane constants of the dense pass
    alignas(16) int4 tlane[32];           // per-lane constants of the chunked time-domain pass (non-run kernels)
    unsigned int next_item;
    alignas(8) unsigned long long mbar;   // completion barrier of the TMA prefetch
};

template <int R1, int R2, int G>
inline size_t fast_fixed_bytes() { return sizeof(FastFixed<R1, R2, G>); }
template <int R1, int R2, int G>
inline size_t fast_smem_bytes(int step, int blob_words, bool runs)
{
    using S = FastShape<R1, R2, G>;
    const size_t span_max = size_t(G - 1) * step + S::N;
    // see the kernel: with run staging the carried tail must survive, otherwise the whole span is dead after pass 1
    const bool zs_alias = runs ? size_t(G) * step >= 2 * size_t(G) * S::ZS : span_max >= 2 * size_t(G) * S::ZS;
    const size_t nrun = (span_max / 8 + 4) & ~size_t(3);
    return fast_fixed_bytes<R1, R2, G>() + sizeof(int) * ((blob_words + 3) & ~3) + 2 * sizeof(float) * nrun +
           sizeof(float) * (span_max + 8) + (zs_alias ? 0 : sizeof(float2) * G * S::ZS) +
           (runs ? sizeof(short) * (size_t(G) * step + 16) : 0);
}

// RAGGED (row modes only): every clip takes its own row counts from p.len (ragged_rows); a template flag so that the
// uniform launches keep their code.
template <int R1, int R2, int G, bool STEP_EVEN, bool RUNS, int MODE, bool RAGGED = false>
__global__ void __launch_bounds__(fast_threads(G), B200AA_FAST_MINBLOCKS) st_fast_kernel(const StParams p, const float2 *__restrict__ g_tw,
                                                                const float2 *__restrict__ g_twp, unsigned int *work_counter)
{
    using S = FastShape<R1, R2, G>;
    constexpr int Nc = S::Nc, N = S::N, K = S::K, Kp = S::Kp, ES = S::ES, H = S::H, ZS = S::ZS, TPF = S::TPF;
    constexpr int NT = fast_threads(G);
    static_assert(NT == S::NT, "one warp per frame slot");
    static_assert(NT >= S::FftThreads && NT >= 16 * G + 32, "transform threads, and at least one warp next to the dense pass");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int step = p.step;
    // shared-memory layout: all fixed-size arrays sit at compile-time offsets (no address arithmetic to keep
    // live in registers); the three arrays whose size depends on the hop come last
    using Fixed = FastFixed<R1, R2, G>;
    Fixed &sm = *reinterpret_cast<Fixed *>(smem_raw);
    float2 *const E = sm.E, *const s_tw = sm.tw, *const s_twp = sm.twp;
    float *const Xprev = sm.Xprev, *const fvrows = sm.fvrows, *const mscr = sm.mscr, *const chr = sm.chr;
    float *const parts = sm.parts;
    int *const blob_s = reinterpret_cast<int *>(smem_raw + sizeof(Fixed));
    const int blob_pad = (p.bl.words + 3) & ~3;
    const int nrun = ((G - 1) * step + N) / 8 + 4 & ~3;
    using runf_t = int;                                                               // sign-flip word of a run
    float *const runE = reinterpret_cast<float *>(blob_s + blob_pad);                 // run partials (RUNS only)
    runf_t *const runF = reinterpret_cast<runf_t *>(runE + nrun);
    float *const sS = reinterpret_cast<float *>(runF + nrun);                         // sample span
    auto TW = [&](int i) -> float2 { return s_tw[i]; };
    auto TWP = [&](int i) -> float2 { return s_twp[i]; };
    // published second-pass outputs [G][ZS]: the float samples of the G frames are dead once pass 1 has read them
    // (with run staging only the tail that the next step reuses must survive; without it the time-domain rows are
    // produced right after staging), so Zs lives on top of them
    const bool zs_alias = RUNS ? (G * step >= 2 * G * ZS) : ((G - 1) * step + N >= 2 * G * ZS);
    float2 *const Zs = zs_alias ? reinterpret_cast<float2 *>(sS)
                                : reinterpret_cast<float2 *>(sS + (((G - 1) * step + N + 8) & ~3));
    // raw int16 landing zone of the TMA prefetch (RUNS only): 8 predecessor samples + G*step new samples
    short *const raw = reinterpret_cast<short *>(sS + (((G - 1) * step + N + 8) & ~3) + (zs_alias ? 0 : 2 * G * ZS));
    float *Xrows = reinterpret_cast<float *>(E);                             // rows f -> Xrows + f*Kp (aliases E)
    static_assert(size_t(G) * Kp * sizeof(float) <= size_t(G) * R1 * ES * sizeof(float2), "alias");
    static_assert((G & (G - 1)) == 0, "tile mapping");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < p.bl.words; i += NT) blob_s[i] = p.blob[i];
    for (int i = tid; i < R1 * R2; i += NT) s_tw[i] = g_tw[i];
    for (int i = tid; i < Nc / 2 + 1; i += NT) s_twp[i] = g_twp[i];
    __syncthreads();
    const int *const blob_t = blob_s;
    const SmallTables tb = bind_tables(blob_t, p.bl);
    if (tid < 32) sm.tlane[tid] = time_lane_init(N, tid);
    if (MODE == kModeFeatures && tid < 16) *reinterpret_cast<int4 *>(sm.dlane + tid * 4) = pair_lane_init<K>(tid);   // dense pass only
    for (int i = tid; i < 2 * Kp; i += NT) Xprev[i] = 0.f;
    if (RUNS && tid == 0) mbar_init(&sm.mbar, 1);
    unsigned tma_phase = 0;       // parity of the next completion to wait for
    __syncthreads();
    const bool fft_thread = tid < S::FftThreads;
    const int ff = tid / TPF, fj = tid - ff * TPF;      // frame slot / index within the frame's TPF threads

    // work items are handed out dynamically (one atomic per item) so the tail of the launch is one item long
    for (int64_t item = blockIdx.x; item < p.n_items;) {
        if (tid == 0) sm.next_item = atomicAdd(work_counter, 1u) + gridDim.x;
        do {
        const int64_t b = item / p.segs_per_clip, seg = item % p.segs_per_clip;
        const int64_t len = p.len ? p.len[b] : p.n_samples;
        // features: frames of the clip; spectrogram / chromagram: the rows of this launch (rows >= n_valid are zero)
        typedef int fidx_t;          // frame / row indices inside a clip fit 32 bits (checked on the host)
        int64_t rows_b = p.rows_launch, valid_b = p.rows_valid;
        if constexpr (RAGGED) ragged_rows<MODE>(p, b, rows_b, valid_b);
        const fidx_t T = fidx_t(MODE == kModeFeatures ? (len < N ? 0 : (len - N) / step + 1) : rows_b);
        const fidx_t n_valid = MODE == kModeFeatures ? T : fidx_t(valid_b);
        const fidx_t t0 = fidx_t(seg * p.seg_len);
        if (t0 >= T) break;
        const fidx_t t1 = (t0 + fidx_t(p.seg_len)) < T ? (t0 + fidx_t(p.seg_len)) : T;
        const b200aa_clip_norm nm = p.norm[b];
        const char *clip = reinterpret_cast<const char *>(p.sig) +
                           size_t(b) * p.clip_stride * (p.dtype == B200AA_DTYPE_I16 ? 2 : 4);
        const SampleReader rd{clip, p.dtype, nm.m};
        const int halo = MODE == kModeFeatures ? int(t0 < 2 ? t0 : 2) : 0;
        // 16-byte loads need the clip base and the step's first sample aligned (8 samples of int16)
        const bool vec_ok = (reinterpret_cast<uintptr_t>(clip) & 15) == 0 && (p.dtype == B200AA_DTYPE_I16 || (step % 4 == 0));

        int fbase = 0;        // ring row that holds the previous frame's features
        bool prefetched = false;   // this step's new samples were fetched by TMA during the previous step
        int xsel = 0;         // which half of Xprev holds the previous step's last |X|
        for (fidx_t g0 = t0 - halo; g0 < t1; g0 += G) {
            const int nrow = int((t1 - g0) < G ? (t1 - g0) : G);          // rows / frames of this step
            // frames that exist (spectrogram / chromagram allocate more rows than their loops fill)
            const int ng = int((n_valid - g0) < nrow ? ((n_valid - g0) > 0 ? (n_valid - g0) : 0) : nrow);
            if (MODE != kModeFeatures && ng < nrow) {
                // zero rows (all threads; rows are disjoint from the ones written below)
                const int width = MODE == kModeSpectrogram ? K : 12;
                for (int e = tid; e < (nrow - ng) * width; e += NT) {
                    const int f = ng + e / width, k = e % width;
                    p.out[(size_t(b) * p.rows_launch + g0 + f) * width + k] = 0.f;
                }
                if (ng == 0) continue;
            }
            // ---- stage the sample span of this step as float (x - m)
            const int span = (ng - 1) * step + N;
            const int64_t sbase = frame_first<MODE>(N, step, g0);
            if (RUNS) {
                // samples shared with the previous step are already converted: move them to the front
                int keep = 0;
                if (g0 > t0 - halo && step < N) {
                    keep = N - step;                       // previous step was a full one (G frames)
                    // up to 2 float4 + 1 run partial per thread (keep <= N - 8 samples)
                    float4 cv[2];
                    float ce[1]; runf_t cf[1];
                    const int src = G * step;
                    static_assert((2 * Nc) / 4 <= 2 * NT && (2 * Nc) / 8 <= NT, "carry copy mapping");
#pragma unroll
                    for (int u = 0; u < 2; ++u)
                        if (tid + u * NT < keep / 4) cv[u] = *reinterpret_cast<const float4 *>(sS + src + 4 * (tid + u * NT));
                    if (tid < keep / 8) { ce[0] = runE[src / 8 + tid]; cf[0] = runF[src / 8 + tid]; }
                    __syncthreads();
#pragma unroll
                    for (int u = 0; u < 2; ++u)
                        if (tid + u * NT < keep / 4) *reinterpret_cast<float4 *>(sS + 4 * (tid + u * NT)) = cv[u];
                    if (tid < keep / 8) { runE[tid] = ce[0]; runF[tid] = cf[0]; }
                }
                if (prefetched) {
                    mbar_wait(&sm.mbar, tma_phase);
                    tma_phase ^= 1u;
                    for (int r = keep / 8 + tid; r < span / 8; r += NT)
                        stage_run_smem(raw + 8 + 8 * (r - keep / 8), true, nm, sS + 8 * r, runE + r, runF + r);
                } else {
                    for (int r = keep / 8 + tid; r < span / 8; r += NT)
                        stage_run(clip, p.dtype, vec_ok, sbase + 8 * r, nm, sS + 8 * r, runE + r, runF + r);
                }
            } else {
                for (int i = tid; i < span; i += NT) sS[i] = rd(sbase + i);
            }
            __syncthreads();
            if (!RUNS && MODE == kModeFeatures) {
                // hops that are not whole 8-sample runs: time-domain rows straight from the staged samples, one warp
                // per frame, BEFORE the FFT (pass 2 reuses the sample buffer)
                for (int f = warp; f < ng; f += G) {
                    int ru = fbase + 1 + f;
                    if (ru > G) ru -= G + 1;
                    const float *frs = sS + f * step;
                    time_features_chunked([&](int n) { return frs[n]; }, N, nm, sm.tlane[lane], parts + warp * 64, fvrows + ru * kFvStride, lane);
                }
            }
            // ---- TMA: fetch the next step's new samples (same work item) while this step computes
            prefetched = false;
            if (RUNS && MODE == kModeFeatures && p.dtype == B200AA_DTYPE_I16 && vec_ok && step < N && g0 + G < t1) {
                const fidx_t gn = g0 + G;
                const int ngn = int((t1 - gn) < G ? (t1 - gn) : G);
                const int keepn = N - step;
                const int cnt = (ngn - 1) * step + N - keepn;                    // new samples of that step
                const short *src = reinterpret_cast<const short *>(clip) + (frame_first<MODE>(N, step, gn) + keepn - 8);
                if (tid == 0) tma_load_1d(raw, src, unsigned(cnt + 8) * 2u, &sm.mbar);
                prefetched = true;
            }

            // ---- pass 1: thread (frame ff, column n2 = fj): R1-point FFT over n1 of z[R2*n1 + n2], twiddle, transpose
            float d0 = 0.f;                 // first sample of the frame (kept for the DC bin)
            if (fft_thread && ff < ng && fj < R2) {
                const float *fr = sS + ff * step;
                d0 = fr[0];
                float2 v1[R1];
#pragma unroll
                for (int n1 = 0; n1 < R1; ++n1) {
                    float2 z;
                    if (STEP_EVEN) z = *reinterpret_cast<const float2 *>(fr + 2 * (R2 * n1 + fj));
                    else { z.x = fr[2 * (R2 * n1 + fj)]; z.y = fr[2 * (R2 * n1 + fj) + 1]; }
                    v1[n1] = make_float2(z.x - d0, z.y - d0);
                }
                fft_r<R1>(v1);
                float2 *Ef = E + size_t(ff) * R1 * ES;
#pragma unroll
                for (int k1 = 0; k1 < R1; ++k1) {
                    const float2 w = k1 == 0 ? make_float2(1.f, 0.f) : TW(k1 * R2 + fj);
                    Ef[k1 * ES + fj] = k1 == 0 ? v1[0] : cmul(v1[k1], w);
                }
            }
            __syncthreads();
            // ---- pass 2: thread (frame ff, row k1 = fj): R2-point FFT over n2 -> Z[k1 + R1*k2]
            float2 v[R2];
            if (fft_thread && ff < ng && fj < R1) {
                const float2 *Ef = E + size_t(ff) * R1 * ES + fj * ES;
#pragma unroll
                for (int n2 = 0; n2 < R2; ++n2) v[n2] = Ef[n2];
                fft_r<R2>(v);
                float2 *Zf = Zs + size_t(ff) * ZS;
#pragma unroll
                for (int k2 = H; k2 < R2; ++k2) Zf[fj + R1 * (k2 - H)] = v[k2];
            }
            __syncthreads();    // all E reads done (|X| rows alias E) and partner values visible
            // ---- post-process: X[k] = ev + W_N^k od, X[Nc-k] = conj(ev - W_N^k od) from (Z[k], Z[Nc-k])
            if (fft_thread && ff < ng && fj < R1) {
                const float2 *Zf = Zs + size_t(ff) * ZS;
                float *Xf = Xrows + size_t(ff) * Kp;
                const float sc = nm.a / float(2 * K);
                auto pair = [&](int k, float2 zk, bool do_mirror) {
                    const float2 zp = Zf[(Nc - k) - R1 * H];
                    const float2 ev = make_float2(zk.x + zp.x, zk.y - zp.y);
                    const float2 od = make_float2(zk.y + zp.y, zp.x - zk.x);
                    const float2 t = cmul(od, TWP(k));
                    const float ar = ev.x + t.x, ai = ev.y + t.y;
                    const float br = ev.x - t.x, bi = ev.y - t.y;
                    Xf[k] = fsqrt_pos(fmaf(ar, ar, ai * ai)) * sc;
                    if (do_mirror) Xf[Nc - k] = fsqrt_pos(fmaf(br, br, bi * bi)) * sc;
                };
#pragma unroll
                for (int k2 = 0; k2 < H; ++k2) {
                    const int k = fj + R1 * k2;
                    if (k2 == 0 && fj == 0) {
                        // DC: a * sum(d - d0) + N * (a*d0 + bp)
                        Xf[0] = fabsf(fmaf(nm.a, v[0].x + v[0].y, float(N) * fmaf(nm.a, d0, nm.bp))) / float(K);
                    } else {
                        pair(k, v[k2], true);
                    }
                }
                {   // middle index k2 = H: only the lower partner of each pair computes it
                    const int k = fj + R1 * H;
                    if (2 * k < Nc) pair(k, v[H], true);
                    else if (2 * k == Nc) {          // self-paired bin Nc/2 (R even, thread 0): |X| = |Z|
                        Xf[k] = fsqrt_pos(fmaf(v[H].x, v[H].x, v[H].y * v[H].y)) * (2.f * sc);
                    }
                }
            }
            for (int e = tid; e < G * (Kp - K); e += NT) {     // zero padding of the rows (bins K .. Kp-1)
                const int f = e / (Kp - K), i = e - f * (Kp - K);
                Xrows[size_t(f) * Kp + K + i] = 0.f;
            }
            __syncthreads();

            if constexpr (MODE == kModeSpectrogram) {
                // rows are contiguous in the output: consecutive threads -> consecutive bins
                float *dst = p.out + (size_t(b) * p.rows_launch + g0) * K;
                for (int e = tid; e < ng * K; e += NT) {
                    const int f = e / K, k = e - f * K;
                    dst[e] = Xrows[size_t(f) * Kp + k];
                }
                __syncthreads();
                continue;
            } else if constexpr (MODE == kModeChromagram) {
                for (int f = warp; f < ng; f += G) {
                    const float *X = Xrows + size_t(f) * Kp;
                    float sxx = 0.f;
#pragma unroll
                    for (int i = 0; i < DenseShape<K>::C; ++i) { const float v = X[lane * DenseShape<K>::C + i]; sxx = fmaf(v, v, sxx); }
                    sxx = warp_sum(sxx);
                    const float ch = chroma_lane(X, sxx, tb, lane);
                    if (lane < 12) p.out[(size_t(b) * p.rows_launch + g0 + f) * 12 + lane] = ch;
                }
                __syncthreads();
                continue;
            }
            // ---- phase A: lower half of the CTA = dense spectral rows (two frames per warp); upper half = mel taps +
            // log10 and the raw chroma sums of all frames
            const int half = lane >> 4, l16 = lane & 15;
            const int wv = warp < G / 2 ? warp : warp - G / 2;
            const int fq = 2 * wv + half;
            const bool act = fq < ng;
            const int f = act ? fq : 0;                         // inactive halves shadow frame 0 (no stores)
            int rr = fbase + 1 + f;
            if (rr > G) rr -= G + 1;
            float *fv = fvrows + rr * kFvStride;
            if (warp >= G / 2) {
                upper_mel_chroma<G, NT - 16 * G>(Xrows, Kp, ng, tb, blob_t + p.bl.mel_grp, mscr, chr, tid - 16 * G);
            } else {
                const fidx_t fr = g0 + f;
                const float *X = Xrows + size_t(f) * Kp;
                const bool has_prev = (fr > 0) && !(f == 0 && g0 == t0 - halo);
                const float *Xp = has_prev ? (f > 0 ? Xrows + size_t(f - 1) * Kp : Xprev + xsel * Kp) : X;
                // the neighbour's row sum is produced concurrently by another half-warp: recompute it in the same order
                const float rs = row_sum_h<K>(Xp, l16);
                const float sxp = (has_prev && f == 0) ? fvrows[fbase * kFvStride + 34] : rs;
                spectral_features_h<K>(X, Xp, sxp, sm.dlane + l16 * 4, parts + (warp * 2 + half) * 32, fv, l16, act,
                                       (act && f == ng - 1) ? Xprev + (xsel ^ 1) * Kp : nullptr);
            }
            __syncthreads();
            // ---- phase B: DCT rows (all threads), then chroma normalisation (lower half) / time-domain rows (upper half)
            flat_dct<G, NT>(mscr, ng, tb, fvrows, fbase, tid);
            if (warp >= G / 2) {
                if (RUNS) {
                    // the NT/32 - G/2 upper warps take the frames two at a time (one round when every frame pair has a warp)
                    constexpr int UW = NT / 32 - G / 2;
                    static_assert((G / 2) % UW == 0, "whole rounds over the frame pairs");
#pragma unroll
                    for (int rd = 0; rd < (G / 2) / UW; ++rd) {
                        const int fq2 = 2 * (wv + rd * UW) + half;
                        const bool act2 = fq2 < ng;
                        const int f2 = act2 ? fq2 : 0;
                        int r2 = fbase + 1 + f2;
                        if (r2 > G) r2 -= G + 1;
                        time_features_runs_h<N>(runE + (f2 * step) / 8, runF + (f2 * step) / 8, fvrows + r2 * kFvStride, l16, act2);
                    }
                }
            } else {
                chroma_finalize_h(chr + f * 12, fv, l16, act);
            }
            __syncthreads();
            // ---- store the [n_out x 8] tile: 8 consecutive threads -> 8 consecutive frames of one feature row
            float *const out_b = p.out + size_t(b) * p.n_out * p.t_stride + g0;
            for (int e = tid; e < p.n_out * G; e += NT) {
                const int f = e / G, c = e % G;
                const fidx_t fr = g0 + c;
                if (c >= ng || fr < t0) continue;
                int r1 = fbase + 1 + c;
                if (r1 > G) r1 -= G + 1;
                int r0 = fbase + c;
                if (r0 > G) r0 -= G + 1;
                float val;
                if (f < B200AA_N_BASE) val = fvrows[r1 * kFvStride + f];
                else {
                    const int fb = f - B200AA_N_BASE;
                    val = fr == 0 ? 0.f : fvrows[r1 * kFvStride + fb] - fvrows[r0 * kFvStride + fb];
                }
                out_b[size_t(f) * p.t_stride + c] = val;
            }
            // the last frame of this step becomes "previous" for the next one: advance the ring / flip the buffer
            // (no copies, no barrier: the next step's writers of these arrays run several barriers later)
            fbase += ng;
            if (fbase > G) fbase -= G + 1;
            xsel ^= 1;
        }
        } while (0);
        __syncthreads();
        item = sm.next_item;
        __syncthreads();
    }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
// window -> (R1, R2) of the register-tiled transform (window = 2 * R1 * R2); 0 = use the generic kernel
inline bool fast_shape_for_window(int window, int *r1, int *r2)
{
    switch (window) {
    case 800: *r1 = 20; *r2 = 20; return true;     // 50 ms @ 16 kHz
    case 882: *r1 = 21; *r2 = 21; return true;     // 20 ms @ 44.1 kHz
    case 400: *r1 = 20; *r2 = 10; return true;     // 50 ms @ 8 kHz, 25 ms @ 16 kHz
    case 480: *r1 = 20; *r2 = 12; return true;     // 30 ms @ 16 kHz, 10 ms @ 48 kHz
    case 600: *r1 = 20; *r2 = 15; return true;     // 75 ms @ 8 kHz
    case 320: *r1 = 16; *r2 = 10; return true;     // 20 ms @ 16 kHz, 40 ms @ 8 kHz
    case 640: *r1 = 20; *r2 = 16; return true;     // 40 ms @ 16 kHz
    default: return false;
    }
}

inline int fast_plan_init(int window, FastTables *ft, int *kind)
{
    *kind = 0;
    int R1 = 0, R2 = 0;
    if (!fast_shape_for_window(window, &R1, &R2)) return B200AA_OK;
    const int Nc = R1 * R2, N = 2 * Nc;
    if (b200aa_host::upload(b200aa_host::twiddle_grid(R1, R2, Nc), ft->tw) != cudaSuccess ||
        b200aa_host::upload(b200aa_host::twiddles(Nc / 2 + 1, N), ft->twp) != cudaSuccess)
        return B200AA_ERR_CUDA;
    ft->R = R1 * 100 + R2;
    *kind = ft->R;
    return B200AA_OK;
}

#ifndef B200AA_LAYOUT_ONLY     // tests/smem_budget_host.cu includes this header for the layout arithmetic only
template <int R1, int R2, int G, bool EVEN, bool RUNS, int MODE>
inline int fast_launch_t(const FastTables &ft, StParams p, int sm_count, int64_t T, unsigned int *ctr, cudaStream_t st)
{
    constexpr int NT = fast_threads(G);
    const size_t smem = fast_smem_bytes<R1, R2, G>(p.step, p.bl.words, RUNS);
    if (smem > 110u * 1024u) return B200AA_ERR_UNSUPPORTED;      // very large hop: leave it to the generic kernel
    auto kern = st_fast_kernel<R1, R2, G, EVEN, RUNS, MODE>;
    if constexpr (MODE != kModeFeatures) {
        if (p.len) kern = st_fast_kernel<R1, R2, G, EVEN, RUNS, MODE, true>;
    }
    int occ = 1;
    if (resident_ctas(kern, NT, smem, 110 * 1024, occ) != cudaSuccess) return B200AA_ERR_CUDA;
    const int64_t slots = int64_t(sm_count) * occ;
    // work items: >= ~8 per CTA slot for balance, as long as possible to amortise the 2-frame halo, and
    // seg + 2 a multiple of the 8-frame CTA step so no step runs half empty
    int64_t per_clip = (slots * 8 + p.n_clips - 1) / p.n_clips;
    if (per_clip < 1) per_clip = 1;
    int64_t seg = (T + per_clip - 1) / per_clip;
    // throughput runs keep items >= 46 frames (halo <= 4 %); when the whole launch cannot fill the machine anyway
    // (a single short clip through the NumPy drop-in) latency wins: one 8-frame CTA step per item
    const int64_t min_seg = (T * p.n_clips >= 46 * slots) ? 46 : 6;
    if (seg < min_seg) seg = min_seg;
    seg = ((seg + 2 + G - 1) / G) * G - 2;
    if (seg > T) seg = T;
    p.seg_len = seg;
    p.segs_per_clip = (T + seg - 1) / seg;
    p.n_items = p.segs_per_clip * p.n_clips;
    if (p.n_items >= (int64_t(1) << 31) || T >= (int64_t(1) << 31)) return B200AA_ERR_UNSUPPORTED;   // 32-bit work / frame indices
    const int64_t grid = p.n_items < slots ? p.n_items : slots;
    if (getenv("B200AA_DEBUG"))
        fprintf(stderr, "[b200aa] fast kernel %dx%d G=%d runs=%d mode=%d: smem %zu B, %d CTAs/SM, grid %lld, %lld items of %lld frames\n",
                R1, R2, G, int(RUNS), MODE, smem, occ, (long long)grid, (long long)p.n_items, (long long)seg);
    if (cudaMemsetAsync(ctr, 0, sizeof(unsigned int), st) != cudaSuccess) return B200AA_ERR_CUDA;
    kern<<<(unsigned)grid, NT, smem, st>>>(p, static_cast<const float2 *>(ft.tw.get()), static_cast<const float2 *>(ft.twp.get()), ctr);
    return cudaPeekAtLastError() == cudaSuccess ? B200AA_OK : B200AA_ERR_CUDA;    // the caller fetches (and clears) the text
}

// run staging needs whole 8-sample runs per frame, per entropy block (window % 80 == 0) and per hop.  Every frame starts
// at a multiple of the step, or of the step past the (even; with runs, multiple of 8) window.
template <int R1, int R2, int MODE>
inline int fast_launch_shape(const FastTables &ft, const StParams &p, int sm_count, int64_t T, unsigned int *ctr, cudaStream_t st)
{
    constexpr int G = B200AA_FAST_G;
    constexpr int N = 2 * R1 * R2;
    const bool even = (p.step % 2) == 0;
    if (N % 80 == 0) {
        const bool runs = (p.step % 8) == 0 && (p.clip_stride % 8) == 0;
        if (runs) return fast_launch_t<R1, R2, G, true, N % 80 == 0, MODE>(ft, p, sm_count, T, ctr, st);
    }
    return even ? fast_launch_t<R1, R2, G, true, false, MODE>(ft, p, sm_count, T, ctr, st)
                : fast_launch_t<R1, R2, G, false, false, MODE>(ft, p, sm_count, T, ctr, st);
}

template <int MODE>
inline int fast_launch_mode(int kind, const FastTables &ft, const StParams &p, int sm_count, int64_t T, unsigned int *ctr, cudaStream_t st)
{
    switch (kind) {
    case 2020: return fast_launch_shape<20, 20, MODE>(ft, p, sm_count, T, ctr, st);
    case 2121: return fast_launch_shape<21, 21, MODE>(ft, p, sm_count, T, ctr, st);
    case 2010: return fast_launch_shape<20, 10, MODE>(ft, p, sm_count, T, ctr, st);
    case 2012: return fast_launch_shape<20, 12, MODE>(ft, p, sm_count, T, ctr, st);
    case 2015: return fast_launch_shape<20, 15, MODE>(ft, p, sm_count, T, ctr, st);
    case 1610: return fast_launch_shape<16, 10, MODE>(ft, p, sm_count, T, ctr, st);
    case 2016: return fast_launch_shape<20, 16, MODE>(ft, p, sm_count, T, ctr, st);
    default: return B200AA_ERR_UNSUPPORTED;
    }
}
#endif  // B200AA_LAYOUT_ONLY

}  // namespace b200aa
