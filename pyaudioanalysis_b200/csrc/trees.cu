// libb200aa.so -- Tree-ensemble classification (kernel 8).
#include <algorithm>
#include <memory>

#include "../../include/b200aa.h"
#include "entry.h"
#include "trees.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 8: tree-ensemble classification, bit for bit scikit-learn's predict / predict_proba (csrc/trees.cuh)
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(b200aa_tree_node) == sizeof(trees::Node), "node layout of the C ABI");

struct b200aa_trees {
    int device;
    int64_t n_nodes, n_leaves;
    int n_trees, n_classes, n_feats, mode, allow_nan;
    void *blob;                         // [nodes | roots | values | init] on `device`
    const trees::Node *nodes;
    const int32_t *roots;
    const double *values, *init;
};

namespace {
constexpr int kTreeWarps = 4;           // warps per CTA of trees_kernel, one query row per warp at a time
}  // namespace

// One warp per query row (grid-stride).  The row, cast to float32, goes to shared memory; lane j walks tree t0 + j of
// each block of 32 trees and leaves its leaf row in shared memory; then lane c adds class c's leaf values of the block in
// tree order, so every class sum is the sequential sum over the trees.  Per warp: [x: F floats | 32 leaves | C sums].
template <class Tq>
__global__ void __launch_bounds__(kTreeWarps * 32) trees_kernel(const trees::Node *__restrict__ nodes,
                                                               const int32_t *__restrict__ roots, int n_trees,
                                                               const double *__restrict__ values,
                                                               const double *__restrict__ init, int mode, int C, int F,
                                                               bool allow_nan, const Tq *__restrict__ q, int64_t n,
                                                               int64_t stride, int64_t *__restrict__ ids,
                                                               double *__restrict__ scores, int32_t *__restrict__ bad)
{
    extern __shared__ __align__(16) unsigned char trees_smem[];
    const int w = threadIdx.x / 32, lane = threadIdx.x % 32;
    const size_t per = trees::warp_bytes(F, C);
    float *x = reinterpret_cast<float *>(trees_smem + w * per);
    int32_t *leaf = reinterpret_cast<int32_t *>(x + F);
    double *acc = reinterpret_cast<double *>(trees_smem + w * per + per - size_t(C) * sizeof(double));
    for (int64_t row = int64_t(blockIdx.x) * kTreeWarps + w; row < n; row += int64_t(gridDim.x) * kTreeWarps) {
        bool b = false;
        for (int j = lane; j < F; j += 32) x[j] = trees::cast(q[row * stride + j], allow_nan, b);
        b = __any_sync(0xffffffffu, b);
        for (int c = lane; c < C; c += 32) acc[c] = init ? init[c] : 0.0;
        __syncwarp();
        for (int t0 = 0; t0 < n_trees; t0 += 32) {
            const int nt = min(32, n_trees - t0);
            if (lane < nt) leaf[lane] = trees::walk(nodes, roots[t0 + lane], x);
            __syncwarp();
            for (int c = lane; c < C; c += 32) {
                double a = acc[c];
                for (int j = 0; j < nt; ++j) {
                    const int tc = trees::tree_class(mode, t0 + j, C);
                    if (tc < 0) a = trees::dadd(a, values[int64_t(leaf[j]) * C + c]);
                    else if (tc == c) a = trees::dadd(a, values[leaf[j]]);
                }
                acc[c] = a;
            }
            __syncwarp();
        }
        double best = 0.0, s0 = 0.0;
        int bi = -1;
        for (int c = lane; c < C; c += 32) {
            const double s = trees::finish(mode, acc[c], n_trees);
            scores[row * C + c] = s;
            if (c == 0) s0 = s;
            if (bi < 0 || trees::better(s, c, best, bi)) { best = s; bi = c; }
        }
        for (int off = 16; off > 0; off >>= 1) {
            const double ob = __shfl_down_sync(0xffffffffu, best, off);
            const int oi = __shfl_down_sync(0xffffffffu, bi, off);
            if (oi >= 0 && (bi < 0 || trees::better(ob, oi, best, bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            ids[row] = trees::class_id(mode, C, s0, bi);
            bad[row] = b ? 1 : 0;
        }
        __syncwarp();
    }
}

extern "C" int b200aa_trees_create(b200aa_trees **out, const b200aa_tree_node *h_nodes, int64_t n_nodes,
                                   const int32_t *h_roots, int n_trees, const double *h_values, int64_t n_leaves,
                                   int n_classes, int n_feats, int mode, const double *h_init, int allow_nan)
{
    if (!out) return B200AA_ERR_INVALID;
    *out = nullptr;
    REFUSE_CAPTURE(nullptr, "b200aa_trees_create", kWhyAllocates);
    if (!h_nodes || !h_roots || !h_values || n_nodes < 1 || n_nodes > INT32_MAX || n_trees < 1 || n_leaves < 1 ||
        n_leaves > INT32_MAX || n_classes < 1 || n_feats < 1 || (mode != trees::kForestMean && mode != trees::kBoostSum) ||
        (mode == trees::kBoostSum && !h_init))
        return B200AA_ERR_INVALID;
    if (h_roots[0] != 0) return B200AA_ERR_INVALID;
    // every tree a contiguous node range whose children come after their parent inside it: walks stay in the range and end
    for (int t = 0; t < n_trees; ++t) {
        const int64_t lo = h_roots[t], hi = t + 1 < n_trees ? h_roots[t + 1] : n_nodes;
        if (hi <= lo || hi > n_nodes) return B200AA_ERR_INVALID;
        for (int64_t i = lo; i < hi; ++i) {
            const b200aa_tree_node &nd = h_nodes[i];
            if (nd.left < 0) {
                if (nd.right < 0 || nd.right >= n_leaves) return B200AA_ERR_INVALID;
            } else {
                const int f = nd.feature & trees::kFeatureMask;
                if (nd.left <= i || nd.left >= hi || nd.right <= i || nd.right >= hi || f >= n_feats) return B200AA_ERR_INVALID;
            }
        }
    }
    if (trees::warp_bytes(n_feats, n_classes) * kTreeWarps > 48 * 1024) return B200AA_ERR_UNSUPPORTED;
    const size_t vals = size_t(n_leaves) * (mode == trees::kForestMean ? size_t(n_classes) : 1);
    const bool has_init = mode == trees::kBoostSum;         // a forest's sums start at 0: h_init is not read
    Layout L;
    const size_t nodes_at = L.add(size_t(n_nodes) * sizeof(trees::Node)), roots_at = L.add(size_t(n_trees) * sizeof(int32_t)),
                 values_at = L.add(vals * sizeof(double)), init_at = L.add(has_init ? size_t(n_classes) * sizeof(double) : 0);
    std::unique_ptr<b200aa_trees> m(new b200aa_trees{});
    CK(cudaGetDevice(&m->device));
    CK(cudaMalloc(&m->blob, L.bytes()));
    char *base = static_cast<char *>(m->blob);
    // The upload goes through a stream of its own and is waited for, so the model is on the device when create returns:
    // a copy from pageable memory may return before its DMA lands, and a caller's non-blocking stream is not ordered
    // after the legacy default stream.
    cudaStream_t up = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(base + nodes_at, h_nodes, size_t(n_nodes) * sizeof(trees::Node), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(base + roots_at, h_roots, size_t(n_trees) * sizeof(int32_t), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(base + values_at, h_values, vals * sizeof(double), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess && has_init)
        e = cudaMemcpyAsync(base + init_at, h_init, size_t(n_classes) * sizeof(double), cudaMemcpyHostToDevice, up);
    if (up) {
        const cudaError_t es = cudaStreamSynchronize(up);
        if (e == cudaSuccess) e = es;
        cudaStreamDestroy(up);
    }
    if (e != cudaSuccess) {
        cudaFree(m->blob);
        return cuda_fail(e, "upload (tree ensemble)");
    }
    m->n_nodes = n_nodes;
    m->n_leaves = n_leaves;
    m->n_trees = n_trees;
    m->n_classes = n_classes;
    m->n_feats = n_feats;
    m->mode = mode;
    m->allow_nan = allow_nan ? 1 : 0;
    m->nodes = Layout::at<const trees::Node>(base, nodes_at);
    m->roots = Layout::at<const int32_t>(base, roots_at);
    m->values = Layout::at<const double>(base, values_at);
    m->init = has_init ? Layout::at<const double>(base, init_at) : nullptr;
    *out = m.release();
    return B200AA_OK;
}

extern "C" int b200aa_trees_destroy(b200aa_trees *model)
{
    if (!model) return B200AA_OK;
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e == cudaSuccess && cur != model->device) e = cudaSetDevice(model->device);
    // work queued on any stream may still read the model
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaFree(model->blob);
    if (cur != model->device) cudaSetDevice(cur);
    delete model;
    return e == cudaSuccess ? B200AA_OK : cuda_fail(e, "cudaFree (tree ensemble)");
}

extern "C" int b200aa_trees_classify(const b200aa_trees *model, const void *d_query, int dtype, int64_t n_query,
                                     int n_feats, int64_t q_stride, int64_t *d_ids, double *d_scores, int32_t *d_bad,
                                     void *stream)
{
    NvtxRange nvtx_("b200aa_trees_classify");
    REFUSE_CAPTURE(stream, "b200aa_trees_classify", "kernel 8 is not captured; call it eagerly");
    if (!model || !d_query || !d_ids || !d_scores || !d_bad || n_query < 0 || n_feats != model->n_feats ||
        q_stride < n_feats || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (n_query == 0) return B200AA_OK;
    int cur = 0;
    CK(cudaGetDevice(&cur));
    if (cur != model->device) return B200AA_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = trees::warp_bytes(model->n_feats, model->n_classes) * kTreeWarps;
    const unsigned blocks = unsigned(std::min<int64_t>((n_query + kTreeWarps - 1) / kTreeWarps, INT32_MAX));
    with_real_type(dtype, [&](auto t) {
        trees_kernel<<<blocks, kTreeWarps * 32, smem, st>>>(model->nodes, model->roots, model->n_trees, model->values,
                                                            model->init, model->mode, model->n_classes, model->n_feats,
                                                            model->allow_nan != 0, static_cast<const decltype(t) *>(d_query),
                                                            n_query, q_stride, d_ids, d_scores, d_bad);
    });
    CK_LAUNCH("trees_kernel");
    return B200AA_OK;
}
