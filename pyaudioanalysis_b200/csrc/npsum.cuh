// Correctly rounded double operations and NumPy's pairwise summation, shared by the kernels that reproduce a NumPy
// computation bit for bit (beat.cuh, knn.cuh, hmm.cuh).  __host__ __device__: the host test programs run the same code.
//
// dadd / dsub / dmul / ddiv are the _rn intrinsics on the device: no FMA contraction, and no division expanded into an FMA
// sequence.
#pragma once
#include <cmath>
#include <cstdint>

namespace b200aa {
namespace npy {

constexpr int kLeaf = 128;              // NumPy's PW_BLOCKSIZE

__host__ __device__ inline double dadd(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline double dsub(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
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
__host__ __device__ inline double ddiv(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

__host__ __device__ inline double dsqrt(double a)
{
#ifdef __CUDA_ARCH__
    return __dsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}

// np.add.reduce of get(off) .. get(off + n - 1): NumPy's pairwise summation.  Below 8 elements a running sum from 0.0; up to
// 128, eight running accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added in sequence; above 128,
// a split at n/2 rounded down to a multiple of 8.  Elements at index >= nz are +0.0 and are not read: the sums here are of
// values >= +0.0 (or NaN), for which x + 0.0 == x, so a subtree lying entirely at or beyond nz sums to +0.0 whatever its shape.
// With nz = off + n every element is read and the sum is NumPy's for values of any sign.
template <class G>
__host__ __device__ double pairwise_sum(const G &get, int64_t off, int64_t n, int64_t nz)
{
    if (n <= 0 || off >= nz) return 0.0;
    auto at = [&](int64_t i) { return i < nz ? get(i) : 0.0; };
    if (n < 8) {
        double r = 0.0;
        for (int64_t i = 0; i < n; ++i) r = dadd(r, at(off + i));
        return r;
    }
    if (n <= kLeaf) {
        double r[8];
        for (int j = 0; j < 8; ++j) r[j] = at(off + j);
        int64_t i = 8;
        for (; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; ++j) r[j] = dadd(r[j], at(off + i + j));
        double res = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
        for (; i < n; ++i) res = dadd(res, at(off + i));
        return res;
    }
    int64_t n2 = n / 2;
    n2 -= n2 % 8;
    return dadd(pairwise_sum(get, off, n2, nz), pairwise_sum(get, off + n2, n - n2, nz));
}

// The subtree of pairwise_sum(n) that lane k of 2^levels lanes sums: `levels` splits, taken along k's bits from the top.  A leaf
// reached early stays with the leftmost lane below it; the other lanes get an empty range.  Combining the lane sums as
// s[k] = s[k] + s[k + 2^j] for j = 0 .. levels - 1 (k a multiple of 2^(j+1)) then reproduces the tree: a split node adds its
// halves left + right, and a leaf adds only +0.0s.
__host__ __device__ inline void pairwise_part(int64_t n, int levels, int k, int64_t &off, int64_t &len)
{
    off = 0;
    len = n;
    for (int j = levels - 1; j >= 0; --j) {
        const int bit = (k >> j) & 1;
        if (len > kLeaf) {
            int64_t n2 = len / 2;
            n2 -= n2 % 8;
            if (bit) { off += n2; len -= n2; } else { len = n2; }
        } else if (bit) {
            len = 0;
        }
    }
}

}  // namespace npy
}  // namespace b200aa
