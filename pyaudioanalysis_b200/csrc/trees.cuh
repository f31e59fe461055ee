// Tree-ensemble classification (kernel 8): scikit-learn 1.9's predict / predict_proba of RandomForestClassifier,
// ExtraTreesClassifier and GradientBoostingClassifier for a matrix of query rows, bit for bit:
//   input     every value cast to float32 (round to nearest, subnormals kept); a value that is or becomes +-inf, or a NaN
//             where the model refuses NaN, flags the row (scikit-learn raises ValueError for it);
//   walk      NaN goes to the missing side of the node, otherwise left iff x <= threshold (tree/_tree.pyx, _apply_dense);
//   forest    P[c] = (((0 + v_0[c]) + v_1[c]) + ...) / n_trees in tree order (ensemble/_forest.py), id the first maximum;
//   boosting  raw[k] = init[k] + v_k(stage 0) + v_k(stage 1) + ... in stage order, every v already scaled by the learning
//             rate on the host (ensemble/_gradient_boosting.pyx); id raw >= 0 for K = 1, else the first maximum.
// The pieces are __host__ __device__: tests/trees_host.cu runs them on the CPU.
//
// Node thresholds are stored as float32: for float32 x and finite float64 t, x <= t <=> x <= RD_f32(t) (t rounded toward
// -inf), so the host rounds every threshold down and the walk compares two floats.
#pragma once
#include <cfloat>
#include <cstdint>

#include "npsum.cuh"

namespace b200aa {
namespace trees {

using npy::dadd;
using npy::ddiv;

constexpr int32_t kMissingLeft = int32_t(0x80000000u);     // bit 31 of Node::feature: a NaN goes to the left child
constexpr int32_t kFeatureMask = 0x7fffffff;

enum Mode { kForestMean = 0, kBoostSum = 1 };

// One node of the flattened ensemble (16 bytes).  Internal: left / right are indices into the node array, feature the
// column (with kMissingLeft), threshold RD_f32 of scikit-learn's.  Leaf: left < 0 and right is the leaf's row of values.
struct Node {
    int32_t left, right, feature;
    float threshold;
};
static_assert(sizeof(Node) == 16, "16-byte nodes");

__host__ __device__ inline bool is_nan(float x) { return x != x; }
__host__ __device__ inline bool is_inf(float x) { return x > FLT_MAX || x < -FLT_MAX; }

// float32 value of a query element as validate_data(dtype=np.float32) makes it, and whether it makes the row refused
__host__ __device__ inline float cast(double v, bool allow_nan, bool &bad)
{
#ifdef __CUDA_ARCH__
    const float x = __double2float_rn(v);
#else
    const float x = float(v);
#endif
    if (is_inf(x) || (!allow_nan && is_nan(x))) bad = true;
    return x;
}
__host__ __device__ inline float cast(float x, bool allow_nan, bool &bad)
{
    if (is_inf(x) || (!allow_nan && is_nan(x))) bad = true;
    return x;
}

// shared memory of one warp of the kernel: [the row as float32 (F) | 32 leaf rows | C class sums], the sums 8-aligned
__host__ __device__ inline size_t warp_bytes(int n_feats, int n_classes)
{
    return ((size_t(n_feats) * sizeof(float) + 32 * sizeof(int32_t) + 7) & ~size_t(7)) + size_t(n_classes) * sizeof(double);
}

// one step of the walk: the child a query value goes to
__host__ __device__ inline int32_t child(const Node &nd, float x)
{
    const bool left = is_nan(x) ? (nd.feature & kMissingLeft) != 0 : x <= nd.threshold;
    return left ? nd.left : nd.right;
}

// the leaf row a query row x (float32, after cast) reaches from node `root`
__host__ __device__ inline int32_t walk(const Node *nodes, int32_t root, const float *x)
{
    Node nd = nodes[root];
    while (nd.left >= 0) nd = nodes[child(nd, x[nd.feature & kFeatureMask])];
    return nd.right;
}

// the class a tree's leaf value is added to: every class in a forest (-1), class t mod K in boosting
__host__ __device__ inline int tree_class(int mode, int t, int K) { return mode == kBoostSum ? t % K : -1; }

// the score of a class from its sum: the mean over the trees in a forest, the raw sum in boosting
__host__ __device__ inline double finish(int mode, double sum, int64_t n_trees)
{
    return mode == kForestMean ? ddiv(sum, double(n_trees)) : sum;
}

// np.argmax order: a larger score wins, an equal one keeps the lower class
__host__ __device__ inline bool better(double a, int ia, double b, int ib) { return a > b || (a == b && ia < ib); }

// the class id of a row whose best class is `best`: boosting with K = 1 thresholds its one raw score at 0
__host__ __device__ inline int64_t class_id(int mode, int K, double score0, int best)
{
    return (mode == kBoostSum && K == 1) ? (score0 >= 0.0 ? 1 : 0) : best;
}

}  // namespace trees
}  // namespace b200aa
