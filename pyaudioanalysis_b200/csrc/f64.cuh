// Float64 feature path (kernel family 12): the pieces that make a float64 feature matrix equal to the float64 oracle,
// rows 0 and 1 bit for bit.  __host__ __device__: tests/f64_host.cu runs the same code on the CPU.
//
// Clip normalisation (reference ShortTermFeatures.py:567-570, :14-19; oracle.normalize_clip), bit for bit NumPy:
//   y = x / 32768.0;  mean = np.mean(y) = (0 + pairwise(y)) / n;  y = y - mean;  y = y / (max|y| + 1e-10)
// x / 32768.0 is x * 2^-15: the same real value, so the same correctly rounded double.  The max is exact in any order.
//
// Sums the oracle takes with np.sum are NumPy's pairwise sum (npsum.cuh), split across the 32 lanes of a warp by
// npy::pairwise_part and combined in tree order (lane_pairwise + the combine of the kernels): zcr and energy (rows 0, 1),
// the entropies' block sums, the centroid / spread / flux sums and sum(X^2).  The others follow the oracle's loop flavour
// (oracle/st_oracle.py:169-278) in the order it writes them: np.cumsum is sequential, the chroma fold adds the slots of a
// pitch class in ascending order, and the mel / DCT products (a BLAS dot in the reference, whose order is not fixed) run
// in sequence.
#pragma once
#include <cmath>
#include <cstdint>

#include "../../include/b200aa.h"
#include "front.cuh"
#include "npsum.cuh"

namespace b200aa {
namespace f64 {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsqrt;
using npy::dsub;

constexpr double kEps = 2.220446049250313e-16;     // sys.float_info.epsilon, ShortTermFeatures.py:11
constexpr int kLevels = 5;                         // the pairwise tree split across the 32 lanes of a warp

// x / 32768.0 (exact scaling by a power of two)
__host__ __device__ inline double scaled(double x) { return dmul(x, 1.0 / 32768.0); }

// sample x of the clip, normalised: ((x / 32768) - mean) / (max + 1e-10)
__host__ __device__ inline double normalised(double x, const b200aa_clip_norm_f64 &nm)
{
    return ddiv(dsub(scaled(x), nm.mean), nm.scale);
}

// lane `lane`'s part of NumPy's pairwise sum of get(0) .. get(n - 1) split across 2^levels lanes: its subtree's sum
template <class G>
__host__ __device__ double lane_pairwise(const G &get, int64_t n, int levels, int lane)
{
    int64_t off, len;
    npy::pairwise_part(n, levels, lane, off, len);
    return front::pairwise_flat([&](int64_t i) { return get(off + i); }, len);
}

// np.sum of get(0) .. get(n - 1) on one thread: the lane parts combined in tree order (the host's statement of the
// warp reduction)
template <class G>
__host__ __device__ double np_sum_lanes(const G &get, int64_t n)
{
    double s[1 << kLevels];
    for (int k = 0; k < (1 << kLevels); ++k) s[k] = lane_pairwise(get, n, kLevels, k);
    for (int j = 0; j < kLevels; ++j)
        for (int k = 0; k + (1 << j) < (1 << kLevels); k += 2 << j) s[k] = dadd(s[k], s[k + (1 << j)]);
    return dadd(0.0, s[0]);
}

// np.sign as -1, 0, +1
__host__ __device__ inline int sign_of(double v) { return (v > 0.0) - (v < 0.0); }

// rows 0 and 1 from their sums: zcr = (sum |diff(sign(x))| / 2) / (w - 1.0) (:22-26), energy = sum(x^2) / w (:29-31);
// flips is the integer sum of |diff(sign(x))|, exact in any order
__host__ __device__ inline double zcr_of(int64_t flips, int w) { return ddiv(ddiv(double(flips), 2.0), double(w) - 1.0); }
__host__ __device__ inline double energy_of(double sum_sq, int w) { return ddiv(sum_sq, double(w)); }

// one term -s * log2(s + eps) of an entropy (:34-51, :85-107) before the negation: s = block / (total + eps)
template <class Log2>
__host__ __device__ inline double entropy_term(double block, double total, const Log2 &log2_)
{
    const double s = ddiv(block, dadd(total, kEps));
    return dmul(s, log2_(dadd(s, kEps)));
}

// -np.sum of the 10 entropy terms t[0..9]
__host__ __device__ inline double entropy_of(const double *t)
{
    return -dadd(0.0, front::pairwise_flat([t](int64_t i) { return t[i]; }, 10));
}

// One output of a Stockham pass of radix R over a transform of length Nc (the generic kernel's one-output-per-thread
// form, in fp64): output o of a pass with Ns = product of the earlier radices.  tw[j] = exp(-2 pi i j / Nc).
struct Cplx {
    double x, y;
};
template <class Src, class Tw>
__host__ __device__ inline Cplx stockham_output(const Src &src, int o, int Nc, int Ns, int R, const Tw &tw)
{
    const int NsR = Ns * R, stride = Nc / R, tstep = Nc / NsR;
    const int hi = o / NsR, rem = o - hi * NsR;
    const int q = rem / Ns, k = rem - q * Ns;
    const int j = hi * Ns + k;
    const int ph = int((int64_t(k) * tstep + int64_t(q) * stride) % Nc);
    int idx = 0;
    double ax = 0.0, ay = 0.0;
    for (int r = 0; r < R; ++r) {
        const Cplx t = tw(idx);
        const Cplx v = src(j + r * stride);
        ax = fma(v.x, t.x, fma(-v.y, t.y, ax));
        ay = fma(v.x, t.y, fma(v.y, t.x, ay));
        idx += ph;
        if (idx >= Nc) idx -= Nc;
    }
    return {ax, ay};
}

// |X[k]| / K, as np.abs(...) / K (npy_hypot)
__host__ __device__ inline double magnitude(Cplx z, int K) { return ddiv(hypot(z.x, z.y), double(K)); }

// Mid-term window j of a row of T frames (MidTermFeatures.py:110-126): the Python slice [c0 : min(c0 + ratio, T)]
// (a negative end counts from the end), its np.mean / np.std, and np.nan_to_num of both
__host__ __device__ inline double nan_to_num(double v)
{
    if (v != v) return 0.0;
    if (v - v != v - v) return v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    return v;
}
template <class Row>
__host__ __device__ inline void mid_window(const Row &row, int64_t T, int64_t j, int64_t ratio, int64_t stepr, double &mean,
                                           double &std)
{
    const int64_t c0 = j * stepr;
    int64_t c1 = c0 + ratio < T ? c0 + ratio : T;
    if (c1 < 0) c1 = c1 + T > 0 ? c1 + T : 0;
    const int64_t n = c1 > c0 ? c1 - c0 : 0;
    if (n == 0) {
        mean = std = 0.0;           // 0 / 0 of an empty slice, then nan_to_num
        return;
    }
    front::pool_window([&](int64_t k) { return row(c0 + k); }, n, mean, std);
    mean = nan_to_num(mean);
    std = nan_to_num(std);
}

// The long-term mean of one mid-term row of M windows: mid.T.mean(axis=0) reduces along the row's stride-1 axis, NumPy's
// pairwise sum, then one division (0 / 0 = NaN for no windows)
template <class Row>
__host__ __device__ inline double long_term_mean(const Row &row, int64_t M)
{
    return ddiv(front::np_sum(row, M, true), double(M));
}

}  // namespace f64
}  // namespace b200aa
