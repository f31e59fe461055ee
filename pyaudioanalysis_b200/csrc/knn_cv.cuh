// kNN cross-validation (kernel 6): the model selection of audioTrainTest.evaluate_classifier (reference
// audioTrainTest.py:576-771) for the library's kNN, every (neighbour count, train / test split) problem in one batch.
// Per problem the training rows are standardised as scikit-learn's StandardScaler().fit(X_train) / transform does it,
// then each test row is classified by kernel 5's distance and select kernels (knn.cuh), bit for bit Knn.classify.
//
// StandardScaler (scikit-learn 1.9, dense float64, no weights: _incremental_mean_and_var, _is_constant_feature,
// _handle_zeros_in_scale) per column, over the training rows in the split's order:
//   s = sum x (np.sum over axis 0 of a C-contiguous matrix adds the rows in sequence), mean = (0 + s) / n, T = s / n,
//   c = sum (x - T), q = sum (x - T)^2, var = (q - c^2 / n) / n,
//   scale = 1 where var <= n * eps * var + (n * mean * eps)^2 (a constant column), else sqrt(var);
//   transform: (x - mean) / scale.
// Every double operation goes through the correctly rounded intrinsics (beat.cuh), so nvcc forms no FMA.  These pieces
// are __host__ __device__: tests/knn_cv_host.cu runs them on the CPU against scikit-learn.
#pragma once
#include <cstdint>

#include "knn.cuh"

namespace b200aa {
namespace knn {

constexpr int kFitThreads = 64;         // columns per CTA of the fit-and-gather kernel

struct Scale {
    double mean, scale;
};

// StandardScaler().fit of one column; x(i) is its value in the split's i-th training row, i < n
template <class X>
__host__ __device__ Scale scaler_fit(const X &x, int64_t n)
{
    const double dn = double(n);
    double s = 0.0;
    for (int64_t i = 0; i < n; ++i) s = dadd(s, x(i));
    const double mean = ddiv(dadd(0.0, s), dn);
    const double T = ddiv(s, dn);
    double c = 0.0, q = 0.0;
    for (int64_t i = 0; i < n; ++i) {
        const double t = dsub(x(i), T);
        c = dadd(c, t);
        q = dadd(q, dmul(t, t));
    }
    const double var = ddiv(dsub(q, ddiv(dmul(c, c), dn)), dn);
    constexpr double eps = 2.220446049250313e-16;      // np.finfo(np.float64).eps
    const double drift = dmul(dmul(dn, mean), eps);
    const bool constant = var <= dadd(dmul(dmul(dn, eps), var), dmul(drift, drift));
    return {mean, constant ? 1.0 : dsqrt(var)};
}

// StandardScaler.transform of one value: X -= mean_; X /= scale_
__host__ __device__ inline double standardise(double x, Scale s) { return ddiv(dsub(x, s.mean), s.scale); }

// the class a training row with class index y votes for in a split whose training rows hold C classes (Knn.classify
// counts labels == i for i < C)
__host__ __device__ inline int32_t split_slot(int32_t y, int32_t C) { return y >= 0 && y < C ? y : -1; }

}  // namespace knn
}  // namespace b200aa
