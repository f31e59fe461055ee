// HMM segmentation (kernel 7): the training statistics of audioSegmentation.train_hmm_compute_statistics (reference
// audioSegmentation.py:287-344) and the diagonal-Gaussian Viterbi decode of GaussianHMM(C, "diag").predict(features.T)
// (:489), in the order of double operations NumPy performs on the reference's own array layouts:
//
//   statistics  features[:, idx] is F-contiguous, so mean(axis=1) and std(axis=1) add the class's windows in sequence from
//               +0.0 (a single feature row is contiguous both ways: NumPy then sums it pairwise);
//               mean = sum / n, ssq = sum of (x - mean) * (x - mean) in the same order, std = sqrt(ssq / n);
//   emission    e_t(j) = -0.5 * (K_j + sum_f (x_tf - mu_jf)^2 / var_jf), K_j = F log 2pi + sum_f log var_jf from the host;
//               X = features.T is F-contiguous, so the sum over f runs in sequence from +0.0 (a clip of one window is
//               contiguous both ways: NumPy sums its row pairwise);
//   Viterbi     delta_0(j) = log pi_j + e_0(j); delta_t(j) = max_i(delta_{t-1}(i) + log A_ij) + e_t(j), serial in t; the
//               last state is the first maximum of delta_{T-1}; the backtrack takes, per step, the pair maximum of
//               (delta_{t-1}(i) + log A_i,next, i), i.e. the LAST i of the maximal value (the pair order of hmmlearn's
//               C++ viterbi).  Backpointers store exactly that choice during the forward pass.
//
// Every double operation is a correctly rounded intrinsic (npsum.cuh): no FMA, no device log.  The max is exact, so every
// delta is bit for bit the host restatement's and only exact ties between paths depend on the tie rule above.
// __host__ __device__: tests/hmm_host.cu runs the same code on the CPU.
#pragma once
#include <cmath>
#include <cstdint>

#include "npsum.cuh"

namespace b200aa {
namespace hmm {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsqrt;
using npy::dsub;

constexpr int kMaxStates = 2048;        // the Viterbi warp keeps delta_{t-1} and delta_t in shared memory: 2 x 16 KiB

// NumPy's sum of get(0) .. get(n - 1) over the reference's layout: in sequence from +0.0, or pairwise when `pairwise`
template <class G>
__host__ __device__ double layout_sum(const G &get, int64_t n, bool pairwise)
{
    if (pairwise) return npy::pairwise_sum(get, 0, n, n);
    double s = 0.0;
    for (int64_t i = 0; i < n; ++i) s = dadd(s, get(i));
    return s;
}

struct ClassStats {
    double sum, mean, ssq, std;
};

// one (class, feature): x(i) is the feature of the class's i-th window, in the concatenated order; pairwise when F == 1
template <class X>
__host__ __device__ ClassStats class_stats(const X &x, int64_t n, bool pairwise)
{
    ClassStats r;
    r.sum = layout_sum(x, n, pairwise);
    r.mean = ddiv(r.sum, double(n));
    const double m = r.mean;
    r.ssq = layout_sum([&](int64_t i) { const double d = dsub(x(i), m); return dmul(d, d); }, n, pairwise);
    r.std = dsqrt(ddiv(r.ssq, double(n)));
    return r;
}

// one (window, state): x(f) the window's features, mu / var the state's rows, konst its K_j; pairwise for a one-window clip
template <class X>
__host__ __device__ double emission(const X &x, const double *mu, const double *var, int F, double konst, bool pairwise)
{
    const double s = layout_sum([&](int64_t f) { const double d = dsub(x(f), mu[f]); return ddiv(dmul(d, d), var[f]); }, F,
                                pairwise);
    return dmul(-0.5, dadd(konst, s));
}

// One Viterbi step for state j: delta_t(j) and its backpointer.  prev(i) = delta_{t-1}(i), logA(i) = log A_ij.  The value is
// std::max over the candidates from -inf; the backpointer is their pair maximum (value, i), which keeps the last of equal
// values.
template <class P, class A>
__host__ __device__ double step(const P &prev, const A &logA, int C, double e, int32_t &bp)
{
    double mx = -INFINITY, pv = -INFINITY;
    int32_t pi = 0;
    for (int32_t i = 0; i < C; ++i) {
        const double v = dadd(prev(i), logA(i));
        if (mx < v) mx = v;
        if (pv < v || (!(v < pv) && pi < i)) { pv = v; pi = i; }
    }
    bp = pi;
    return dadd(mx, e);
}

// std::max_element over delta_{T-1}: the first maximum
template <class D>
__host__ __device__ int32_t last_state(const D &delta, int C)
{
    int32_t best = 0;
    for (int32_t i = 1; i < C; ++i)
        if (delta(best) < delta(i)) best = i;
    return best;
}

}  // namespace hmm
}  // namespace b200aa
