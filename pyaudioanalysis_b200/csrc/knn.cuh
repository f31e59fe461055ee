// kNN classification (kernel 5): the library's own classifier, audioTrainTest.Knn.classify (reference audioTrainTest.py:33-49),
// for a matrix of query vectors.  Every output equals the reference's per-vector result bit for bit:
//   distance  sqrt(((x_0 - v_0)^2 + (x_1 - v_1)^2) + ...), a sequential fp64 sum as scipy's cdist(..., 'euclidean') adds it;
//   selection the k smallest keys (distance, training index), NaN after +inf;
//   votes     P[c] = count(slot == c among the selected) / k, the id the first maximum (np.argmax).
// The pieces the result depends on are __host__ __device__: tests/knn_host.cu runs them on the CPU.
//
// Every double operation goes through the correctly rounded intrinsics on the device (npsum.cuh's dadd / dsub / dmul / ddiv
// / dsqrt): nvcc would otherwise contract (x - v) * (x - v) + s into a DFMA, which cdist does not.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "npsum.cuh"

namespace b200aa {
namespace knn {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsub;
using npy::dsqrt;

constexpr int kQ = 64;                  // queries per CTA tile of the distance kernel
constexpr int kT = 64;                  // training rows per CTA tile
constexpr int kF = 16;                  // features staged in shared memory per step
constexpr int kThreads = 256;           // 16 x 16 threads, each a 4 x 4 register tile of distance chains
constexpr int kDigitBits = 8;           // radix select: 8 passes of 256 bins over the 64-bit keys
constexpr int kBins = 1 << kDigitBits;
constexpr int kVoteClasses = 1024;      // classes counted per pass of the vote (more classes: more passes)
constexpr uint64_t kNanKey = 0x7ff8000000000000ull;
constexpr uint64_t kAll = ~0ull;        // threshold key above every key: all N entries selected (k >= N)

// One problem of a launch of the distance and select kernels (kernel 5 runs one, kernel 6 a batch): training rows
// [train0, train0 + N) of the training matrix (and of its slots), queries [q0, q0 + n_q) of the query matrix, keys
// [key0, key0 + n_q * N), results at [out0, out0 + n_q).  Kernel 6 also reads src_train / src_test, the first entries of
// the problem's training / test row indices, and id, its [C, C] count block.
struct Problem {
    int64_t train0, N, q0, n_q, key0, out0, k;
    int64_t src_train, src_test;
    int32_t C;                          // classes voted for
    int32_t id;
};

// one term of the chain: s + (x - v)^2
__host__ __device__ inline double dist_step(double s, double x, double v)
{
    const double d = dsub(x, v);
    return dadd(s, dmul(d, d));
}

// the whole distance of a query x[0..F) to a training row v[0..F)
template <class X, class V>
__host__ __device__ double distance(const X &x, const V &v, int F)
{
    double s = 0.0;                     // 0 + t_0 == t_0 for every t_0 >= +0 or NaN: the same as starting from t_0
    for (int j = 0; j < F; ++j) s = dist_step(s, x(j), v(j));
    return dsqrt(s);
}

// Sort key of a distance: its bits, which order like the values for distances >= +0; every NaN becomes one NaN above
// +inf, and -0 (never produced by the chain) becomes +0.  Ties are broken by the training index outside the key.
__host__ __device__ inline uint64_t key_of(double d)
{
    if (d != d) return kNanKey;
    if (d == 0.0) return 0;
#ifdef __CUDA_ARCH__
    return uint64_t(__double_as_longlong(d));
#else
    uint64_t u;
    std::memcpy(&u, &d, sizeof u);
    return u;
#endif
}

// the total order of the selection: (key, training index)
__host__ __device__ inline bool key_less(uint64_t ka, int64_t ia, uint64_t kb, int64_t ib)
{
    return ka < kb || (ka == kb && ia < ib);
}

// One radix pass of the k-th smallest key.  hist[b] counts the keys that share the prefix found so far and have digit b
// at this pass; `rank` (1-based) is the wanted key's rank among them.  Returns the digit and leaves the rank within it.
__host__ __device__ inline int select_digit(const unsigned *hist, int64_t &rank)
{
    int64_t below = 0;
    for (int b = 0; b < kBins; ++b) {
        if (below + hist[b] >= rank) {
            rank -= below;
            return b;
        }
        below += hist[b];
    }
    return kBins - 1;                   // unreachable while rank <= the number of keys counted
}

// mask of the key bits fixed before the pass that reads the digit at `shift`
__host__ __device__ inline uint64_t prefix_mask(int shift)
{
    return shift + kDigitBits >= 64 ? 0ull : ~0ull << (shift + kDigitBits);
}

// After the radix passes: thr = the k-th smallest key, r = how many entries with key == thr are selected (the r of lowest
// training index).  An entry is selected when its key is below thr, or equal to it and fewer than r equal keys precede it.
__host__ __device__ inline bool selected(uint64_t key, uint64_t thr, int64_t equal_before, int64_t r)
{
    return key < thr || (key == thr && equal_before < r);
}

// P[c] of a class with `count` of the selected entries
__host__ __device__ inline double vote(int64_t count, int64_t k) { return ddiv(double(count), double(k)); }

// np.argmax over the votes: a higher count wins, an equal count keeps the lower class (counts order like the P[c], which
// share the divisor k)
__host__ __device__ inline bool better(int64_t ca, int64_t ia, int64_t cb, int64_t ib) { return ca > cb || (ca == cb && ia < ib); }

}  // namespace knn
}  // namespace b200aa
