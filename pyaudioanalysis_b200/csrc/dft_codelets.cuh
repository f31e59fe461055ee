// Small forward DFT codelets on register arrays (compile-time trigonometry, lane-wise float2 butterflies).
// Shared by the register-tiled kernel (fast_kernel.cuh) and the butterfly passes of the generic kernel.
#pragma once
#include "common.cuh"

namespace b200aa {

// ----------------------------------------------------------------------------------------------
// compile-time trigonometry (exact argument reduction in turns, Taylor series in double)
// ----------------------------------------------------------------------------------------------
constexpr double kCxPi = 3.14159265358979323846264338327950288;

__host__ __device__ constexpr double cx_sin_small(double x)   // |x| <= pi/2
{
    double x2 = x * x, term = x, sum = x;
    for (int i = 1; i < 16; ++i) { term *= -x2 / double((2 * i) * (2 * i + 1)); sum += term; }
    return sum;
}
__host__ __device__ constexpr double cx_cos_small(double x)
{
    double x2 = x * x, term = 1.0, sum = 1.0;
    for (int i = 1; i < 16; ++i) { term *= -x2 / double((2 * i - 1) * (2 * i)); sum += term; }
    return sum;
}
// cos / sin of 2*pi*p/q
__host__ __device__ constexpr double cx_cos_turn(long p, long q)
{
    p %= q; if (p < 0) p += q;
    if (2 * p > q) p = q - p;                 // cos(2 pi (1 - r)) = cos(2 pi r)
    if (4 * p > q) return -cx_cos_small(2.0 * kCxPi * double(q - 2 * p) / double(2 * q));   // cos(pi - y) = -cos y
    return cx_cos_small(2.0 * kCxPi * double(p) / double(q));
}
__host__ __device__ constexpr double cx_sin_turn(long p, long q)
{
    p %= q; if (p < 0) p += q;
    double sign = 1.0;
    if (2 * p > q) { p = q - p; sign = -1.0; }            // sin(2 pi (1 - r)) = -sin(2 pi r)
    if (4 * p > q) return sign * cx_sin_small(2.0 * kCxPi * double(q - 2 * p) / double(2 * q));   // sin(pi - y) = sin y
    return sign * cx_sin_small(2.0 * kCxPi * double(p) / double(q));
}

template <int P>
struct Trig { float c[P], s[P]; };
template <int P>
__host__ __device__ constexpr Trig<P> make_trig()
{
    Trig<P> t{};
    for (int j = 0; j < P; ++j) { t.c[j] = float(cx_cos_turn(j, P)); t.s[j] = float(cx_sin_turn(j, P)); }
    return t;
}
__host__ __device__ constexpr int cx_modinv(int a, int m)
{
    a %= m;
    for (int x = 1; x < m; ++x) if ((a * x) % m == 1) return x;
    return 1;
}

// ----------------------------------------------------------------------------------------------
// small forward DFTs on register arrays
// ----------------------------------------------------------------------------------------------
// Lane-wise (re, im) arithmetic: f2add / f2sub / f2mul / f2fma, each with one rounding per lane; a float first operand of
// f2mul / f2fma multiplies both lanes.  sm_90 has no packed FP32x2 instructions, so each helper is two scalar FP32
// instructions; on the device they are the explicitly rounded intrinsics, which nvcc never contracts across helpers (a
// product from f2mul is rounded before the f2add that consumes it).
// (the codelets are __host__ __device__ so that tests/test_codelets_cpu.py can run them on the CPU with plain arithmetic)
__host__ __device__ __forceinline__ float2 f2add(float2 a, float2 b)
{
#ifdef __CUDA_ARCH__
    return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#else
    return make_float2(a.x + b.x, a.y + b.y);
#endif
}
__host__ __device__ __forceinline__ float2 f2sub(float2 a, float2 b)
{
#ifdef __CUDA_ARCH__
    return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
#else
    return make_float2(a.x - b.x, a.y - b.y);
#endif
}
__host__ __device__ __forceinline__ float2 f2mul(float2 a, float2 b)
{
#ifdef __CUDA_ARCH__
    return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
#else
    return make_float2(a.x * b.x, a.y * b.y);
#endif
}
__host__ __device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c)
{
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__host__ __device__ __forceinline__ float2 f2mul(float c, float2 a) { return f2mul(make_float2(c, c), a); }
__host__ __device__ __forceinline__ float2 f2fma(float c, float2 a, float2 acc) { return f2fma(make_float2(c, c), a, acc); }

template <int RA, int RB> __host__ __device__ __forceinline__ void fft_pfa(float2 (&v)[RA * RB]);
template <int RA, int RB> __host__ __device__ __forceinline__ void fft_ct(float2 (&v)[RA * RB]);

template <int P>
__host__ __device__ __forceinline__ void dft_small(float2 (&x)[P])
{
    if constexpr (P == 6) {
        fft_pfa<2, 3>(x);                                   // composite factors of the longer codelets (30 = 5 x 6)
    } else if constexpr (P == 8) {
        fft_ct<2, 4>(x);                                    // 32 = 4 x 8
    } else if constexpr (P == 2) {
        const float2 a = x[0], b = x[1];
        x[0] = f2add(a, b); x[1] = f2sub(a, b);
    } else if constexpr (P == 4) {
        const float2 a = f2add(x[0], x[2]), b = f2sub(x[0], x[2]), c = f2add(x[1], x[3]), d = f2sub(x[1], x[3]);
        x[0] = f2add(a, c);
        x[2] = f2sub(a, c);
        x[1] = make_float2(b.x + d.y, b.y - d.x);      // b - i d
        x[3] = make_float2(b.x - d.y, b.y + d.x);      // b + i d
    } else {
        // odd prime: y_k = x0 + sum_j [ (x_j + x_{P-j}) cos(2 pi j k / P) - i (x_j - x_{P-j}) sin(2 pi j k / P) ]
        constexpr Trig<P> T = make_trig<P>();
        constexpr int H = (P - 1) / 2;
        float2 sp[H], dr[H], y[P];
#pragma unroll
        for (int j = 1; j <= H; ++j) {
            sp[j - 1] = f2add(x[j], x[P - j]);
            // -i (x_j - x_{P-j}) = (dy, -dx): kept rotated so the odd part is a plain packed accumulate
            dr[j - 1] = make_float2(x[j].y - x[P - j].y, x[P - j].x - x[j].x);
        }
        y[0] = x[0];
#pragma unroll
        for (int j = 0; j < H; ++j) y[0] = f2add(y[0], sp[j]);
#pragma unroll
        for (int k = 1; k <= H; ++k) {
            float2 re = x[0], im = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 1; j <= H; ++j) {
                const float c = T.c[(j * k) % P], sn = T.s[(j * k) % P];
                re = f2fma(c, sp[j - 1], re);
                im = f2fma(sn, dr[j - 1], im);
            }
            y[k] = f2add(re, im);
            y[P - k] = f2sub(re, im);
        }
#pragma unroll
        for (int k = 0; k < P; ++k) x[k] = y[k];
    }
}

// prime-factor FFT of length RA*RB (coprime), natural order in, natural order out
template <int RA, int RB>
__host__ __device__ __forceinline__ void fft_pfa(float2 (&v)[RA * RB])
{
    constexpr int N = RA * RB;
    float2 U[N];
#pragma unroll
    for (int a = 0; a < RA; ++a) {
        float2 t[RB];
#pragma unroll
        for (int b = 0; b < RB; ++b) t[b] = v[(RB * a + RA * b) % N];
        dft_small<RB>(t);
#pragma unroll
        for (int b = 0; b < RB; ++b) U[a * RB + b] = t[b];
    }
    constexpr int ca = RB * cx_modinv(RB, RA), cb = RA * cx_modinv(RA, RB);
#pragma unroll
    for (int kb = 0; kb < RB; ++kb) {
        float2 t[RA];
#pragma unroll
        for (int a = 0; a < RA; ++a) t[a] = U[a * RB + kb];
        dft_small<RA>(t);
#pragma unroll
        for (int ka = 0; ka < RA; ++ka) v[(ka * ca + kb * cb) % N] = t[ka];
    }
}


// Cooley-Tukey FFT of length RA*RB with compile-time twiddles (needed when the factors are not coprime:
// 16 = 4 x 4).  n = RB*a + b, k = ka + RA*kb.
template <int RA, int RB>
__host__ __device__ __forceinline__ void fft_ct(float2 (&v)[RA * RB])
{
    constexpr int N = RA * RB;
    constexpr Trig<N> T = make_trig<N>();
    float2 U[N];
#pragma unroll
    for (int b = 0; b < RB; ++b) {
        float2 t[RA];
#pragma unroll
        for (int a = 0; a < RA; ++a) t[a] = v[RB * a + b];
        dft_small<RA>(t);
#pragma unroll
        for (int ka = 0; ka < RA; ++ka) {
            const int e = (b * ka) % N;                 // twiddle W_N^(b ka) = cos - i sin
            float2 r = t[ka];
            if (e != 0) {
                if (4 * e == N) r = make_float2(t[ka].y, -t[ka].x);                  // multiply by -i
                else if (2 * e == N) r = make_float2(-t[ka].x, -t[ka].y);
                else if (4 * e == 3 * N) r = make_float2(-t[ka].y, t[ka].x);        // multiply by +i
                else {
                    const float c = T.c[e], sn = -T.s[e];                            // (c + i sn), sn = -sin
                    r = make_float2(fmaf(t[ka].x, c, -t[ka].y * sn), fmaf(t[ka].x, sn, t[ka].y * c));
                }
            }
            U[b * RA + ka] = r;
        }
    }
#pragma unroll
    for (int ka = 0; ka < RA; ++ka) {
        float2 t[RB];
#pragma unroll
        for (int b = 0; b < RB; ++b) t[b] = U[b * RA + ka];
        dft_small<RB>(t);
#pragma unroll
        for (int kb = 0; kb < RB; ++kb) v[ka + RA * kb] = t[kb];
    }
}

// the R-point transforms of the register-tiled kernel (fast_kernel.cuh) and their factorisations
template <int R> struct RFactors;
template <> struct RFactors<10> { static constexpr int A = 2, B = 5; };
template <> struct RFactors<12> { static constexpr int A = 4, B = 3; };
template <> struct RFactors<15> { static constexpr int A = 3, B = 5; };
template <> struct RFactors<20> { static constexpr int A = 4, B = 5; };
template <> struct RFactors<21> { static constexpr int A = 3, B = 7; };
template <> struct RFactors<16> { static constexpr int A = 4, B = 4; };   // not coprime: Cooley-Tukey
template <> struct RFactors<25> { static constexpr int A = 5, B = 5; };   // Cooley-Tukey
template <> struct RFactors<32> { static constexpr int A = 4, B = 8; };   // Cooley-Tukey (8 = 2 x 4)
template <> struct RFactors<30> { static constexpr int A = 5, B = 6; };   // prime-factor (6 = 2 x 3)

template <int R>
__host__ __device__ __forceinline__ void fft_r(float2 (&v)[R])
{
    if constexpr (R == 16 || R == 25 || R == 32) fft_ct<RFactors<R>::A, RFactors<R>::B>(v);   // factors not coprime: Cooley-Tukey
    else fft_pfa<RFactors<R>::A, RFactors<R>::B>(v);                          // prime-factor (twiddle-free)
}

// ----------------------------------------------------------------------------------------------
// 32-point forward FFT in "two sequences per register pair" form (pair kernel, pass 2).
// Input: re[m] = (Re x[2m], Re x[2m+1]), im[m] = (Im x[2m], Im x[2m+1]), m < 16 -- the .x halves are the even-indexed
// samples, the .y halves the odd-indexed ones.  Both 16-point sub-transforms run in the same float2 operations
// (identical twiddles, real constants broadcast to both halves; multiplying by -i is a swap of roles, not an
// instruction), then X[k] = E[k] + W32^k O[k], X[k+16] = E[k] - W32^k O[k] in scalar FMAs.  ~280 instructions
// instead of ~440 for the generic (re, im)-packed Cooley-Tukey codelet.
// ----------------------------------------------------------------------------------------------
struct Soa2 { float2 re, im; };      // one complex element of each of the two sequences

__host__ __device__ __forceinline__ void soa_dft4(Soa2 &x0, Soa2 &x1, Soa2 &x2, Soa2 &x3)
{
    const float2 ar = f2add(x0.re, x2.re), ai = f2add(x0.im, x2.im), br = f2sub(x0.re, x2.re), bi = f2sub(x0.im, x2.im);
    const float2 cr = f2add(x1.re, x3.re), ci = f2add(x1.im, x3.im), dr = f2sub(x1.re, x3.re), di = f2sub(x1.im, x3.im);
    x0.re = f2add(ar, cr); x0.im = f2add(ai, ci);
    x2.re = f2sub(ar, cr); x2.im = f2sub(ai, ci);
    x1.re = f2add(br, di); x1.im = f2sub(bi, dr);        // b - i d
    x3.re = f2sub(br, di); x3.im = f2add(bi, dr);        // b + i d
}
// x *= W_Q^e = cos(2 pi e / Q) - i sin(2 pi e / Q), compile-time e
template <int Q, int E>
__host__ __device__ __forceinline__ void soa_twiddle(Soa2 &x)
{
    constexpr int e = E % Q;
    if constexpr (e == 0) {
    } else if constexpr (4 * e == Q) {              // -i
        const float2 t = x.re; x.re = x.im; x.im = make_float2(-t.x, -t.y);
    } else {
        constexpr float wr = float(cx_cos_turn(e, Q)), wi = float(-cx_sin_turn(e, Q));
        const float2 r = f2fma(-wi, x.im, f2mul(wr, x.re));
        const float2 i = f2fma(wr, x.im, f2mul(wi, x.re));
        x.re = r; x.im = i;
    }
}
__host__ __device__ __forceinline__ void fft32_soa(const float2 (&re)[16], const float2 (&im)[16], float2 (&out)[32])
{
    Soa2 t[16];
#pragma unroll
    for (int m = 0; m < 16; ++m) { t[m].re = re[m]; t[m].im = im[m]; }
    // 16 = 4 x 4, m = 4 a + b, k = ka + 4 kb: four DFT4 over a, twiddle W16^(b ka), four DFT4 over b
#pragma unroll
    for (int b = 0; b < 4; ++b) soa_dft4(t[b], t[4 + b], t[8 + b], t[12 + b]);            // t[4 ka + b]
    soa_twiddle<16, 1>(t[4 + 1]); soa_twiddle<16, 2>(t[8 + 1]); soa_twiddle<16, 3>(t[12 + 1]);
    soa_twiddle<16, 2>(t[4 + 2]); soa_twiddle<16, 4>(t[8 + 2]); soa_twiddle<16, 6>(t[12 + 2]);
    soa_twiddle<16, 3>(t[4 + 3]); soa_twiddle<16, 6>(t[8 + 3]); soa_twiddle<16, 9>(t[12 + 3]);
#pragma unroll
    for (int ka = 0; ka < 4; ++ka) soa_dft4(t[4 * ka], t[4 * ka + 1], t[4 * ka + 2], t[4 * ka + 3]);   // -> E/O[ka + 4 kb] at t[4 ka + kb]
    // radix-2 combination of the even (.x) and odd (.y) transforms
    constexpr Trig<32> T = make_trig<32>();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const int ka = k & 3, kb = k >> 2;
        const Soa2 v = t[4 * ka + kb];
        const float er = v.re.x, ei = v.im.x, orr = v.re.y, oi = v.im.y;
        if (k == 0) {
            out[0] = make_float2(er + orr, ei + oi);
            out[16] = make_float2(er - orr, ei - oi);
        } else if (k == 8) {                         // W = -i: t = (oi, -or)
            out[8] = make_float2(er + oi, ei - orr);
            out[24] = make_float2(er - oi, ei + orr);
        } else {
            const float c = T.c[k], sn = T.s[k];     // W32^k = c - i sn:  t = (or c + oi sn, oi c - or sn)
            out[k] = make_float2(fmaf(oi, sn, fmaf(orr, c, er)), fmaf(-orr, sn, fmaf(oi, c, ei)));
            out[k + 16] = make_float2(fmaf(-oi, sn, fmaf(-orr, c, er)), fmaf(orr, sn, fmaf(-oi, c, ei)));
        }
    }
}

}  // namespace b200aa
