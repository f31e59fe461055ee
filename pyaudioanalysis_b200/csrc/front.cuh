// Scaler, outlier rule and per-frame pooling (kernel 11): the host steps of speaker_diarization and music_thumbnailing
// between the features and the quadratic kernels (9 and 10), bit for bit scikit-learn 1.9, scipy and NumPy.
//
// StandardScaler().fit_transform of a dense float64 [n, D] matrix (_incremental_mean_and_var, _is_constant_feature,
// _handle_zeros_in_scale; knn_cv.cuh states the arithmetic).  Its column sums are np.sum / np.nansum over axis 0, whose
// order follows the layout: a reduction along the axis of smaller stride (a column-major matrix, or one column) is NumPy's
// pairwise sum of each column; otherwise the rows are added in sequence, knn::scaler_fit's order.  A NaN adds +0.0 in its
// place (np.nansum copies the matrix with NaN set to 0) and is left out of its column's count; the constant-feature test
// uses that count.  An all-NaN column has count 0: its mean, variance and output are NaN, as scikit-learn's.  Every sum
// starts from NumPy's identity, +0.0.
//
// Outlier rule (reference audioSegmentation.py:861-865) of the normalised [M, D] matrix:
//   dist_all = np.sum(squareform(pdist(X.T)), axis=0)    the D x D distances between columns, kernel 9's chain; the column
//                                                        sums of a C-contiguous [D, D] array add its rows in sequence
//   keep = dist_all < 1.1 * np.mean(dist_all)            np.mean: the pairwise sum over D, then one division
//
// Pooling (reference :884-906): for frame i of a [F, T] matrix, w = x[f, i:min(i + r, T)] widened to float64 and
//   mean = np.mean(w) = (0 + pairwise(w)) / n,   std = np.std(w) = sqrt((0 + pairwise((w - mean)^2)) / n).
//
// The pieces are __host__ __device__: tests/front_host.cu runs them on the CPU.
#pragma once
#include <cstdint>

#include "cluster.cuh"
#include "knn_cv.cuh"
#include "npsum.cuh"

namespace b200aa {
namespace front {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsqrt;
using npy::dsub;

constexpr int kOutlierThreads = 256;    // one CTA: the D column sums, then the mean and the flags
constexpr int kMaxFeats = 4096;         // D of the outlier rule: its D x D distances take 128 MiB at most

// npy::pairwise_sum(get, 0, n, n) without recursion, whose depth would outgrow a thread's stack on the device: the leaves
// of the tree at depth leaf_levels(n) (npy::pairwise_part), each as NumPy's leaf (cluster::leaf_lane / leaf_finish), summed
// in order and combined on a stack, each node left + right.
// An empty lane adds +0.0, which can only turn a -0.0 node into +0.0: np_sum's leading +0.0 leaves the same total.
template <class G>
__host__ __device__ double pairwise_leaf(const G &get, int64_t off, int64_t n)
{
    const auto at = [&](int64_t i) { return get(off + i); };
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = cluster::leaf_lane(at, n, j);
    return cluster::leaf_finish(r, at, n);
}
template <class G>
__host__ __device__ double pairwise_flat(const G &get, int64_t n)
{
    if (n <= npy::kLeaf) return pairwise_leaf(get, 0, n);
    const int L = cluster::leaf_levels(n);
    double stack[32];                   // L <= 31: pairwise_part takes an int lane
    int top = 0;
    for (int64_t k = 0; k < (int64_t(1) << L); ++k) {
        int64_t off, len;
        npy::pairwise_part(n, L, int(k), off, len);
        stack[top++] = pairwise_leaf(get, off, len);
        for (int64_t m = k; m & 1; m >>= 1) {
            --top;
            stack[top - 1] = dadd(stack[top - 1], stack[top]);
        }
    }
    return stack[0];
}

// NumPy's sum of get(0) .. get(n - 1): +0.0 plus the pairwise sum, or the sequential sum from +0.0
template <class G>
__host__ __device__ double np_sum(const G &get, int64_t n, bool pairwise)
{
    if (pairwise) return dadd(0.0, pairwise_flat(get, n));
    double s = 0.0;
    for (int64_t i = 0; i < n; ++i) s = dadd(s, get(i));
    return s;
}

__host__ __device__ inline bool is_nan(double x) { return x != x; }
__host__ __device__ inline bool is_inf(double x) { return x - x != x - x && x == x; }

// StandardScaler().fit of one column of n rows, x(i) its value in row i; `pairwise` as above.  Sets `inf` when a value is
// +-inf (scikit-learn refuses the matrix).  A column without NaN summed in sequence is knn::scaler_fit's.
template <class X>
__host__ __device__ knn::Scale scaler_fit(const X &x, int64_t n, bool pairwise, bool &inf)
{
    int64_t count = 0;
    bool any_inf = false;
    for (int64_t i = 0; i < n; ++i) {
        const double v = x(i);
        count += !is_nan(v);
        any_inf |= is_inf(v);
    }
    inf = any_inf;
    if (!pairwise && count == n) return knn::scaler_fit(x, n);
    const double dn = double(count);
    const double s = np_sum([&](int64_t i) { const double v = x(i); return is_nan(v) ? 0.0 : v; }, n, pairwise);
    const double mean = ddiv(dadd(0.0, s), dn);
    const double T = ddiv(s, dn);
    const double c = np_sum([&](int64_t i) { const double t = dsub(x(i), T); return is_nan(t) ? 0.0 : t; }, n, pairwise);
    const double q = np_sum([&](int64_t i) {
        const double t = dsub(x(i), T);
        return is_nan(t) ? 0.0 : dmul(t, t);
    }, n, pairwise);
    const double var = ddiv(dsub(q, ddiv(dmul(c, c), dn)), dn);
    constexpr double eps = 2.220446049250313e-16;      // np.finfo(np.float64).eps
    const double drift = dmul(dmul(dn, mean), eps);
    const bool constant = var <= dadd(dmul(dmul(dn, eps), var), dmul(drift, drift));
    return {mean, constant ? 1.0 : dsqrt(var)};
}

// dist_all[j] of the outlier rule: d(i, j) for i = 0 .. D - 1 in sequence, the diagonal squareform's 0.0
template <class Dist>
__host__ __device__ double column_sum(const Dist &d, int D, int j)
{
    double s = 0.0;
    for (int i = 0; i < D; ++i) s = dadd(s, i == j ? 0.0 : d(i, j));
    return s;
}

// np.mean(dist_all) of D column sums; a column is kept when dist_all[j] < outlier_threshold(mean)
template <class G>
__host__ __device__ double outlier_mean(const G &dist_all, int D)
{
    return ddiv(np_sum(dist_all, D, true), double(D));
}
__host__ __device__ inline double outlier_threshold(double mean) { return dmul(1.1, mean); }

// (np.mean(w), np.std(w)) of the n >= 1 values w(0) .. w(n - 1)
template <class W>
__host__ __device__ void pool_window(const W &w, int64_t n, double &mean, double &std)
{
    const double dn = double(n);
    mean = ddiv(np_sum(w, n, true), dn);
    const double m = mean;
    std = dsqrt(ddiv(np_sum([&](int64_t k) { const double t = dsub(w(k), m); return dmul(t, t); }, n, true), dn));
}

}  // namespace front
}  // namespace b200aa
