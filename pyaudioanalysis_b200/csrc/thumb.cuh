// Music thumbnails (kernel 10): music_thumbnailing's self-similarity matrix, diagonal filter, masked argmax and walk
// (reference audioSegmentation.py:40-55, :1093-1180) for one standardised track X [T, F] (one frame per row), bit for bit
// scipy and NumPy:
//
//   S[i, j]   = 1 - squareform(pdist(X, 'cosine'))[i, j]: 1.0 on the diagonal; for i != j
//               dot(u, v) = (a0 + a1) [+ u_{F-1} v_{F-1} when F is odd], a0 the sequential sum of the even-indexed
//               products, a1 of the odd-indexed ones (scipy's two-accumulator loop, no FMA);
//               c = dot(u, v) / (sqrt(dot(u, u)) * sqrt(dot(v, v))), clipped to copysign(1, c) when |c| > 1;
//               S = 1 - (1 - c).  A zero-norm or NaN frame gives NaN.
//   C[i, j]   = convolve2d(S, eye(m), 'valid')[i, j] = S[i+m-1, j+m-1] + ... + S[i, j], added in that order (the kernel is
//               flipped); NaN when any entry of the m x m box at (i, j) is NaN (the zero kernel entries are multiplied
//               too).  R = T - m + 1 rows and columns, T >= m >= 1.
//   min_sm    = np.min(C), NaN when any entry is NaN.
//   mask      entries with |i - j| < diag_gap (5.0 / short_step), i > j, or a row or column outside [lo, hi) (the
//             reference's limit slices, resolved by Python's slice rules) become min_sm.
//   argmax    the first maximum in row-major order, the first NaN when there is one: the largest key
//             (NaN first, value, lowest flat index), which no reduction order changes.
//   walk      the reference's loop (:1168-1177), at most m steps, strict > (a NaN comparison takes the else branch).
//
// The pieces are __host__ __device__, so tests/thumb_host.cu runs the kernels' own order of operations on the CPU.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "npsum.cuh"

namespace b200aa {
namespace thumb {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsub;

constexpr int kTile = 64;           // frames per side of a similarity tile
constexpr int kF = 16;              // features staged in shared memory per step (even: a step keeps the pairs whole)
constexpr int kThreads = 256;       // 16 x 16 threads, each a 4 x 4 register tile of dot products
constexpr int kFTile = 32;          // outputs per side of a filter tile: 32 x 8 threads, four rows each
constexpr int kMaskThreads = 256;

// One track of a launch: its frames are rows x0 .. x0 + T - 1 of X; S at s0 in the similarity buffer, the NaN windows at
// h0 in theirs, C at c0 in the output; rows and columns outside [lo, hi) are masked.
struct Track {
    int64_t x0, T, R, s0, h0, c0, lo, hi;
};

// scipy's cosine dot product of get(k) = (u_k, v_k) products, k < F
template <class G>
__host__ __device__ double dot(const G &prod, int F)
{
    double a0 = 0.0, a1 = 0.0;
    int k = 0;
    for (; k + 1 < F; k += 2) {
        a0 = dadd(a0, prod(k));
        a1 = dadd(a1, prod(k + 1));
    }
    double r = dadd(a0, a1);
    if (k < F) r = dadd(r, prod(k));
    return r;
}

// S[i, j], i != j, from dot(u, v) and the two row norms sqrt(dot(u, u)), sqrt(dot(v, v))
__host__ __device__ inline double similarity(double d, double nu, double nv)
{
    double c = ddiv(d, dmul(nu, nv));
    if (fabs(c) > 1.0) c = copysign(1.0, c);
    return dsub(1.0, dsub(1.0, c));
}

// C[i, j] of a NaN-free box: the diagonal from k = m - 1 down to 0
template <class G>
__host__ __device__ double diag_sum(const G &S, int64_t i, int64_t j, int m)
{
    double s = S(i + m - 1, j + m - 1);
    for (int k = m - 2; k >= 0; --k) s = dadd(s, S(i + k, j + k));
    return s;
}

__host__ __device__ inline uint64_t bits_of(double x)
{
#ifdef __CUDA_ARCH__
    return uint64_t(__double_as_longlong(x));
#else
    uint64_t b;
    std::memcpy(&b, &x, 8);
    return b;
#endif
}
__host__ __device__ inline double double_of(uint64_t b)
{
#ifdef __CUDA_ARCH__
    return __longlong_as_double(static_cast<long long>(b));
#else
    double x;
    std::memcpy(&x, &b, 8);
    return x;
#endif
}

// the order of the non-NaN doubles as unsigned integers, from 1 (-inf) up; 0 and ~0 stay free for NaN
__host__ __device__ inline uint64_t ordered(double x)
{
    const uint64_t b = bits_of(x);
    return (b >> 63) ? ~b : (b | (uint64_t(1) << 63));
}
__host__ __device__ inline double unordered(uint64_t k)
{
    return double_of((k >> 63) ? (k & ~(uint64_t(1) << 63)) : ~k);
}
// np.min's key: the smallest wins, NaN below everything
constexpr uint64_t kMinNaN = 0;
__host__ __device__ inline uint64_t min_key(double x) { return x != x ? kMinNaN : ordered(x); }
__host__ __device__ inline double min_value(uint64_t k) { return k == kMinNaN ? double_of(0x7ff8000000000000ull) : unordered(k); }
// np.argmax's key: the largest wins, NaN above everything; ties go to the lowest flat index
__host__ __device__ inline uint64_t max_key(double x) { return x != x ? ~uint64_t(0) : ordered(x); }
__host__ __device__ inline bool better(uint64_t k1, int64_t i1, uint64_t k2, int64_t i2)
{
    return k1 > k2 || (k1 == k2 && i1 < i2);
}

// the reference's masks: the band |i - j| < gap (a Python int-float compare, exact below 2^53), the lower triangle, and the
// limit slices
__host__ __device__ inline bool masked(int64_t i, int64_t j, double gap, int64_t lo, int64_t hi)
{
    const int64_t d = i > j ? i - j : j - i;
    return double(d) < gap || i > j || i < lo || j < lo || i >= hi || j >= hi;
}

// the reference's walk from the argmax (r, c) over the masked matrix C [R, R]: out = (i1, i2, j1, j2)
template <class G>
__host__ __device__ void walk(const G &C, int64_t R, int64_t r, int64_t c, int m, int64_t *out)
{
    int64_t i1 = r, i2 = r, j1 = c, j2 = c;
    while (i2 - i1 < m) {
        if (i1 <= 0 || j1 <= 0 || i2 >= R - 2 || j2 >= R - 2) break;
        if (C(i1 - 1, j1 - 1) > C(i2 + 1, j2 + 1)) {
            --i1;
            --j1;
        } else {
            ++i2;
            ++j2;
        }
    }
    out[0] = i1;
    out[1] = i2;
    out[2] = j1;
    out[3] = j2;
}

// upper-triangle tile l (row-major over ti <= tj) of an n x n tile grid
__host__ __device__ inline void upper_tile(int64_t l, int64_t n, int64_t &ti, int64_t &tj)
{
    ti = 0;
    while (l >= n - ti) {
        l -= n - ti;
        ++ti;
    }
    tj = ti + l;
}
__host__ __device__ inline int64_t upper_tiles(int64_t n) { return n * (n + 1) / 2; }

}  // namespace thumb
}  // namespace b200aa
