// libb200aa.so -- Forest training (kernel 13).
#include <algorithm>
#include <vector>

#include "../../include/b200aa.h"
#include "entry.h"
#include "forest.cuh"
#include "front.cuh"
#include "knn_cv.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 13: random forest / extra trees training, bit for bit scikit-learn 1.9's fit (csrc/forest.cuh)
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(b200aa_forest_node) == sizeof(forest::NodeOut), "node layout of the C ABI");

__global__ void forest_cast_kernel(const double *__restrict__ X, int64_t n, int F, int64_t stride, float *__restrict__ out)
{
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n * F; i += int64_t(gridDim.x) * blockDim.x)
        out[i] = __double2float_rn(X[(i / F) * stride + i % F]);
}
__global__ void forest_cast_kernel(const float *__restrict__ X, int64_t n, int F, int64_t stride, float *__restrict__ out)
{
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n * F; i += int64_t(gridDim.x) * blockDim.x)
        out[i] = X[(i / F) * stride + i % F];
}

namespace {

// Argument checks shared by the entry points; each returns false where the entry point returns B200AA_ERR_INVALID.
// class labels in [0, n_classes)
bool valid_labels(const int32_t *y, int64_t n, int n_classes)
{
    for (int64_t i = 0; i < n; ++i)
        if (y[i] < 0 || y[i] >= n_classes) return false;
    return true;
}
// finite regression targets
bool finite_targets(const double *y, int64_t n)
{
    for (int64_t i = 0; i < n; ++i)
        if (!(y[i] - y[i] == 0.0)) return false;
    return true;
}
// bootstrap counts in [0, 2^29]
bool valid_weights(const int32_t *w, int64_t count)
{
    for (int64_t i = 0; i < count; ++i)
        if (w[i] < 0 || w[i] > (1 << 29)) return false;
    return true;
}
// Ragged splits of n_problems problems over rows [0, n): offsets from 0, at least one training row and no fewer than zero
// test rows per problem, every index a row.  No test offsets (test_off NULL): no test rows.
bool valid_splits(int64_t n, int64_t n_problems, const int64_t *train_off, const int32_t *train_idx, const int64_t *test_off,
                  const int32_t *test_idx)
{
    const auto rows_in = [n](const int32_t *idx, int64_t lo, int64_t hi) {
        for (int64_t i = lo; i < hi; ++i)
            if (idx[i] < 0 || idx[i] >= n) return false;
        return true;
    };
    if (train_off[0] != 0 || (test_off && test_off[0] != 0)) return false;
    for (int64_t p = 0; p < n_problems; ++p) {
        if (train_off[p + 1] - train_off[p] < 1 || (test_off && test_off[p + 1] < test_off[p])) return false;
        if (!rows_in(train_idx, train_off[p], train_off[p + 1]) || (test_off && !rows_in(test_idx, test_off[p], test_off[p + 1])))
            return false;
    }
    return true;
}

// One tree's slot of global scratch: its builder's own arrays (the head), then the tail every builder writes: stack
// [n + 1], nodes [2 n - 1], values [(2 n - 1) per_node], meta (node_count, max_depth).
struct Slot {
    size_t stack, nodes, values, meta, bytes;
};
Slot slot_after(size_t head, int64_t n, int per_node)
{
    const int64_t cap = 2 * n - 1;
    Layout A(head);
    Slot S;
    S.stack = A.add(size_t(n + 1) * sizeof(forest::StackRec));
    S.nodes = A.add(size_t(cap) * sizeof(forest::NodeOut));
    S.values = A.add(size_t(cap) * per_node * 8);
    S.meta = A.add(2 * sizeof(int64_t));
    S.bytes = A.bytes();
    return S;
}

// a classification tree's slot
struct TreeLayout {
    size_t samples, tmp, keys;
    Slot s;
};
TreeLayout tree_layout(int64_t n, int C)
{
    Layout A;
    TreeLayout L;
    L.samples = A.add(size_t(n) * 4);
    L.tmp = A.add(size_t(n) * 4);
    L.keys = A.add(size_t(forest::pow2_at_least(n)) * 8);
    L.s = slot_after(A.bytes(), n, C);
    return L;
}

// Thread 0 of a build kernel: the tree's node count and depth to its slot's meta, where read_trees finds them
template <class S>
__device__ void put_meta(char *meta, const S *st)
{
    if (threadIdx.x == 0) {
        int64_t *m = reinterpret_cast<int64_t *>(meta);
        m[0] = st->node_count;
        m[1] = st->max_depth;
    }
}

// trees per launch: as many as keep fixed + their slots under the scratch slice bound, at most n_trees; 0 when not even
// one tree fits.  A regression tree's sort keys take 8 F pow2(n) bytes, so at F = 136 one fits for n up to 131 072.
int64_t trees_per_launch(size_t fixed, size_t per_tree, int64_t n_trees)
{
    if (fixed + per_tree > kScratchSliceBytes) return 0;
    return std::min<int64_t>(n_trees, int64_t((kScratchSliceBytes - fixed) / per_tree));
}

// Where a fit returns its trees: per_node values per node, each tree's node count and depth, and the nodes written so far
struct TreesOut {
    b200aa_forest_node *nodes;
    double *values;
    int per_node;
    int64_t capacity, *node_count;
    int32_t *max_depth;
    int64_t written;
};

// One launch's nt trees (slot i at trees + i * S.bytes) to the host as trees t0 .. t0 + nt - 1, their nodes and values
// after those already written; B200AA_ERR_INVALID when they pass the capacity.  Returns with the copies done, so the
// next launch may reuse the slots.
int read_trees(cudaStream_t st, const char *trees, const Slot &S, int64_t t0, int64_t nt, TreesOut &o)
{
    std::vector<int64_t> meta(size_t(nt) * 2);
    for (int64_t i = 0; i < nt; ++i)
        CK(cudaMemcpyAsync(&meta[size_t(i) * 2], trees + size_t(i) * S.bytes + S.meta, 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int64_t i = 0; i < nt; ++i) {
        const int64_t nc = meta[size_t(i) * 2], t = t0 + i;
        o.node_count[t] = nc;
        o.max_depth[t] = int32_t(meta[size_t(i) * 2 + 1]);
        if (o.written + nc > o.capacity) return B200AA_ERR_INVALID;
        const char *tb = trees + size_t(i) * S.bytes;
        CK(cudaMemcpyAsync(o.nodes + o.written, tb + S.nodes, size_t(nc) * sizeof(forest::NodeOut), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(o.values + o.written * o.per_node, tb + S.values, size_t(nc) * o.per_node * 8,
                           cudaMemcpyDeviceToHost, st));
        o.written += nc;
    }
    CK(cudaStreamSynchronize(st));    // the next launch reuses the scratch the copies read
    return B200AA_OK;
}

// X [n, F] (float32 or float64, rows row_stride apart) to dense float32 Xf, rounded to nearest as fit casts
int cast_to_f32(const void *d_X, int dtype, int64_t n, int F, int64_t row_stride, float *Xf, cudaStream_t st)
{
    const unsigned blocks = unsigned(std::min<int64_t>((n * F + 255) / 256, 4096));
    with_real_type(dtype, [&](auto t) {
        forest_cast_kernel<<<blocks, 256, 0, st>>>(static_cast<const decltype(t) *>(d_X), n, F, row_stride, Xf);
    });
    CK_LAUNCH("forest_cast_kernel");
    return B200AA_OK;
}

}  // namespace

// One CTA per tree of the slice: build_tree with the block as its team.
__global__ void __launch_bounds__(forest::kThreads) forest_build_kernel(const float *__restrict__ X,
                                                                       const int32_t *__restrict__ y, int64_t n, int F,
                                                                       int C, int max_features, int kind,
                                                                       const int32_t *__restrict__ w,
                                                                       const uint32_t *__restrict__ seeds,
                                                                       char *__restrict__ scratch, TreeLayout L)
{
    extern __shared__ __align__(16) unsigned char forest_smem[];
    const forest::Team tm{int(threadIdx.x), int(blockDim.x)};
    char *base = scratch + size_t(blockIdx.x) * L.s.bytes;
    forest::Tree T{X, y, w ? w + int64_t(blockIdx.x) * n : nullptr, n, F, C, max_features, kind,
                   reinterpret_cast<int32_t *>(base + L.samples), reinterpret_cast<int32_t *>(base + L.tmp),
                   reinterpret_cast<uint64_t *>(base + L.keys), reinterpret_cast<forest::StackRec *>(base + L.s.stack),
                   reinterpret_cast<forest::NodeOut *>(base + L.s.nodes), reinterpret_cast<double *>(base + L.s.values)};
    forest::carve_smem(forest_smem, blockDim.x, T);
    forest::build_tree(T, tm, seeds[blockIdx.x]);
    put_meta(base + L.s.meta, T.st);
}

extern "C" int b200aa_forest_fit(const void *d_X, int dtype, int64_t n, int n_feats, int64_t row_stride,
                                 const int32_t *h_y, int n_classes, int kind, int n_trees, int max_features,
                                 const int32_t *h_weights, const uint32_t *h_seeds, b200aa_forest_node *h_nodes,
                                 double *h_values, int64_t node_capacity, int64_t *h_node_count, int32_t *h_max_depth,
                                 void *stream)
{
    NvtxRange nvtx_("b200aa_forest_fit");
    REFUSE_CAPTURE(stream, "b200aa_forest_fit", kWhyHostArrays);
    if (!d_X || !h_y || !h_seeds || !h_nodes || !h_values || !h_node_count || !h_max_depth || n < 1 ||
        n > (int64_t(1) << 29) || n_feats < 1 || row_stride < n_feats || n_classes < 1 || n_trees < 1 ||
        (kind != forest::kBest && kind != forest::kRandom) || max_features < 1 || max_features > n_feats ||
        node_capacity < 0 || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (!valid_labels(h_y, n, n_classes) || (h_weights && !valid_weights(h_weights, int64_t(n_trees) * n)))
        return B200AA_ERR_INVALID;
    if (n_feats > forest::kMaxFeats || n_classes > forest::kMaxClasses) return B200AA_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = forest::smem_bytes(n_feats, n_classes);
    CK(cudaFuncSetAttribute(forest_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(forest::kSmemCap)));
    const TreeLayout L = tree_layout(n, n_classes);
    Layout A;
    const size_t x_at = A.add(size_t(n) * n_feats * 4), y_at = A.add(size_t(n) * 4), seeds_at = A.add(size_t(n_trees) * 4);
    const size_t w_row = h_weights ? align256(size_t(n) * 4) : 0;    // a tree's weights: one padded row per tree
    const int64_t slice = std::max<int64_t>(1, trees_per_launch(A.bytes(), L.s.bytes + w_row, n_trees));    // never refused
    const size_t trees_at = A.add(size_t(slice) * L.s.bytes), w_at = A.add(size_t(slice) * w_row);
    StreamScratch scratch(st);
    int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    float *Xf = Layout::at<float>(base, x_at);
    int32_t *y = Layout::at<int32_t>(base, y_at);
    uint32_t *seeds = Layout::at<uint32_t>(base, seeds_at);
    char *trees = Layout::at<char>(base, trees_at);
    int32_t *w = h_weights ? Layout::at<int32_t>(base, w_at) : nullptr;
    if ((rc = cast_to_f32(d_X, dtype, n, n_feats, row_stride, Xf, st)) != B200AA_OK) return rc;
    CK(cudaMemcpyAsync(y, h_y, size_t(n) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(seeds, h_seeds, size_t(n_trees) * 4, cudaMemcpyHostToDevice, st));
    TreesOut out{h_nodes, h_values, n_classes, node_capacity, h_node_count, h_max_depth, 0};
    for (int64_t t0 = 0; t0 < n_trees; t0 += slice) {
        const int64_t nt = std::min<int64_t>(slice, n_trees - t0);
        if (w) CK(cudaMemcpyAsync(w, h_weights + t0 * n, size_t(nt * n) * 4, cudaMemcpyHostToDevice, st));
        forest_build_kernel<<<unsigned(nt), forest::kThreads, smem, st>>>(Xf, y, n, n_feats, n_classes, max_features, kind,
                                                                         w, seeds + t0, trees, L);
        CK_LAUNCH("forest_build_kernel");
        if ((rc = read_trees(st, trees, L.s, t0, nt, out)) != B200AA_OK) return scratch.done(rc);
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernel 13 in model selection: every (parameter, experiment) problem of evaluate_classifier for the two forests
// ------------------------------------------------------------------------------------------------
// One thread per column: StandardScaler().fit over the problem's training rows in split order (kernel 6's
// knn::scaler_fit), then the training and test rows standardised and cast to float32 as fit / predict cast them.
__global__ void forest_cv_scale_kernel(const double *__restrict__ X, int F, const int32_t *__restrict__ train, int64_t n_train,
                                       const int32_t *__restrict__ test, int64_t n_test, float *__restrict__ Xtr,
                                       float *__restrict__ Xte)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const knn::Scale sc = knn::scaler_fit([&](int64_t i) { return X[int64_t(train[i]) * F + f]; }, n_train);
    for (int64_t i = 0; i < n_train; ++i) Xtr[i * F + f] = __double2float_rn(knn::standardise(X[int64_t(train[i]) * F + f], sc));
    for (int64_t i = 0; i < n_test; ++i) Xte[i * F + f] = __double2float_rn(knn::standardise(X[int64_t(test[i]) * F + f], sc));
}

// One thread per test row: walk every tree of the slice (forest::tree_apply) and add
// its leaf's values to the row's class sums in tree order (forest predict_proba); after the last slice P = sum / T, the
// first maximum is the prediction (classes_.take(argmax)), mapped to its class over all problems and counted.
__global__ void forest_cv_classify_kernel(const float *__restrict__ Xte, int64_t n_test, int F, int C, const char *__restrict__ trees,
                                          Slot S, int nt, bool first, bool last, int n_trees,
                                          double *__restrict__ acc, const int32_t *__restrict__ to_global,
                                          const int32_t *__restrict__ y_test, int n_classes, int32_t *__restrict__ pred,
                                          unsigned long long *__restrict__ counts)
{
    const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= n_test) return;
    const float *x = Xte + r * F;
    double *a = acc + r * C;
    if (first)
        for (int c = 0; c < C; ++c) a[c] = 0.0;
    for (int t = 0; t < nt; ++t) {
        const forest::NodeOut *nodes = reinterpret_cast<const forest::NodeOut *>(trees + size_t(t) * S.bytes + S.nodes);
        const double *values = reinterpret_cast<const double *>(trees + size_t(t) * S.bytes + S.values);
        const int32_t i = forest::tree_apply(nodes, [x](int f) { return x[f]; });
        for (int c = 0; c < C; ++c) a[c] = forest::dadd(a[c], values[int64_t(i) * C + c]);
    }
    if (!last) return;
    double best = 0.0;
    int bi = -1;
    for (int c = 0; c < C; ++c) {
        const double pc = forest::ddiv(a[c], double(n_trees));
        if (bi < 0 || pc > best) {
            best = pc;
            bi = c;
        }
    }
    const int32_t g = to_global[bi];
    pred[r] = g;
    atomicAdd(&counts[int64_t(y_test[r]) * n_classes + g], 1ull);
}

extern "C" int b200aa_forest_cross_validate(const double *d_X, int64_t n, int n_feats, const int32_t *h_y, int n_classes,
                                            int kind, int64_t n_problems, const int64_t *h_train_off,
                                            const int32_t *h_train_idx, const int64_t *h_test_off,
                                            const int32_t *h_test_idx, const int32_t *h_n_trees,
                                            const int32_t *h_weights, const uint32_t *h_seeds, int32_t *d_pred,
                                            int64_t *d_counts, void *stream)
{
    NvtxRange nvtx_("b200aa_forest_cross_validate");
    REFUSE_CAPTURE(stream, "b200aa_forest_cross_validate", kWhyHostArrays);
    if (!d_X || !h_y || !h_train_off || !h_train_idx || !h_test_off || !h_test_idx || !h_n_trees || !h_seeds || !d_pred ||
        !d_counts || n < 1 || n > (int64_t(1) << 29) || n_feats < 1 || n_classes < 1 || n_problems < 1 ||
        (kind != forest::kBest && kind != forest::kRandom) || (kind == forest::kBest) != (h_weights != nullptr))
        return B200AA_ERR_INVALID;
    if (!valid_labels(h_y, n, n_classes) || !valid_splits(n, n_problems, h_train_off, h_train_idx, h_test_off, h_test_idx))
        return B200AA_ERR_INVALID;
    int64_t ntr_max = 0, nte_max = 0, weights_total = 0, t_max = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off[p + 1] - h_test_off[p];
        if (ntr > n || h_n_trees[p] < 1) return B200AA_ERR_INVALID;
        ntr_max = std::max(ntr_max, ntr);
        nte_max = std::max(nte_max, nte);
        t_max = std::max<int64_t>(t_max, h_n_trees[p]);
        weights_total += int64_t(h_n_trees[p]) * ntr;
    }
    if (h_weights && !valid_weights(h_weights, weights_total)) return B200AA_ERR_INVALID;
    if (n_feats > forest::kMaxFeats || n_classes > forest::kMaxClasses) return B200AA_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int C = n_classes, F = n_feats, max_features = forest::sqrt_features(F);
    CK(cudaFuncSetAttribute(forest_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(forest::kSmemCap)));
    // every region sized by the largest problem
    const TreeLayout Lmax = tree_layout(ntr_max, C);
    const int64_t nte1 = std::max<int64_t>(nte_max, 1);
    Layout A;
    const size_t ylocal_at = A.add(size_t(ntr_max) * 4), train_at = A.add(size_t(ntr_max) * 4), test_at = A.add(size_t(nte1) * 4),
                 map_at = A.add(forest::kMaxClasses * 4), xtr_at = A.add(size_t(ntr_max) * F * 4),
                 xte_at = A.add(size_t(nte1) * F * 4), acc_at = A.add(size_t(nte1) * C * 8), seeds_at = A.add(size_t(t_max) * 4),
                 ytest_at = A.add(size_t(nte1) * 4);
    const size_t w_row = h_weights ? align256(size_t(ntr_max) * 4) : 0;    // a tree's weights: one padded row per tree
    const int64_t slice = std::max<int64_t>(1, trees_per_launch(A.bytes(), Lmax.s.bytes + w_row, t_max));    // never refused
    const size_t trees_at = A.add(size_t(slice) * Lmax.s.bytes), w_at = A.add(size_t(slice) * w_row);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    int32_t *d_ylocal = Layout::at<int32_t>(base, ylocal_at), *d_train = Layout::at<int32_t>(base, train_at);
    int32_t *d_test = Layout::at<int32_t>(base, test_at), *d_map = Layout::at<int32_t>(base, map_at);
    float *d_xtr = Layout::at<float>(base, xtr_at), *d_xte = Layout::at<float>(base, xte_at);
    double *d_acc = Layout::at<double>(base, acc_at);
    uint32_t *d_seeds = Layout::at<uint32_t>(base, seeds_at);
    int32_t *d_ytest = Layout::at<int32_t>(base, ytest_at);
    char *d_trees = Layout::at<char>(base, trees_at);
    int32_t *d_w = h_weights ? Layout::at<int32_t>(base, w_at) : nullptr;
    CK(cudaMemsetAsync(d_counts, 0, size_t(n_problems) * C * C * sizeof(int64_t), st));
    std::vector<int32_t> ylocal(ntr_max), ytest(std::max<int64_t>(nte_max, 1)), map(forest::kMaxClasses);
    int64_t tree0 = 0, w0 = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off[p + 1] - h_test_off[p];
        const int32_t *tr = h_train_idx + h_train_off[p], *te = h_test_idx + h_test_off[p];
        const int T = h_n_trees[p];
        // the classifier's classes_: the sorted class indices present in the training rows
        int32_t local_of[forest::kMaxClasses];
        for (int c = 0; c < C; ++c) local_of[c] = -1;
        for (int64_t i = 0; i < ntr; ++i) local_of[h_y[tr[i]]] = 0;
        int Cl = 0;
        for (int c = 0; c < C; ++c)
            if (local_of[c] == 0) {
                local_of[c] = Cl;
                map[Cl++] = c;
            }
        for (int64_t i = 0; i < ntr; ++i) ylocal[i] = local_of[h_y[tr[i]]];
        for (int64_t i = 0; i < nte; ++i) ytest[i] = h_y[te[i]];
        CK(cudaMemcpyAsync(d_train, tr, size_t(ntr) * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_ylocal, ylocal.data(), size_t(ntr) * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_map, map.data(), size_t(Cl) * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_seeds, h_seeds + tree0, size_t(T) * 4, cudaMemcpyHostToDevice, st));
        if (nte) {
            CK(cudaMemcpyAsync(d_test, te, size_t(nte) * 4, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_ytest, ytest.data(), size_t(nte) * 4, cudaMemcpyHostToDevice, st));
        }
        forest_cv_scale_kernel<<<unsigned((F + 63) / 64), 64, 0, st>>>(d_X, F, d_train, ntr, d_test, nte, d_xtr, d_xte);
        CK_LAUNCH("forest_cv_scale_kernel");
        const TreeLayout L = tree_layout(ntr, Cl);
        const size_t smem_p = forest::smem_bytes(F, Cl);
        for (int64_t t0 = 0; t0 < T; t0 += slice) {
            const int64_t nt = std::min<int64_t>(slice, T - t0);
            if (d_w) CK(cudaMemcpyAsync(d_w, h_weights + w0 + t0 * ntr, size_t(nt * ntr) * 4, cudaMemcpyHostToDevice, st));
            forest_build_kernel<<<unsigned(nt), forest::kThreads, smem_p, st>>>(d_xtr, d_ylocal, ntr, F, Cl, max_features, kind,
                                                                               d_w, d_seeds + t0, d_trees, L);
            CK_LAUNCH("forest_build_kernel");
            if (nte) {
                forest_cv_classify_kernel<<<unsigned((nte + 127) / 128), 128, 0, st>>>(
                    d_xte, nte, F, Cl, d_trees, L.s, int(nt), t0 == 0, t0 + nt == T, T, d_acc, d_map, d_ytest, C,
                    d_pred + h_test_off[p], reinterpret_cast<unsigned long long *>(d_counts + p * C * C));
                CK_LAUNCH("forest_cv_classify_kernel");
            }
        }
        tree0 += T;
        w0 += int64_t(T) * ntr;
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernel 13, regression: RandomForestRegressor fit, bit for bit scikit-learn 1.9's (csrc/forest.cuh,
// build_regression_tree), and the forest branch of evaluate_regression's model selection
// ------------------------------------------------------------------------------------------------
namespace {

// a regression tree's slot of at most n samples, from offset `at`
struct RegLayout {
    size_t samples, idx, fv, keys, weights;
    Slot s;
};
RegLayout reg_layout(int64_t n, int F, size_t at = 0)
{
    Layout A(at);
    RegLayout L;
    L.samples = A.add(size_t(n) * 4);
    L.idx = A.add(size_t(n) * 4);
    L.fv = A.add(size_t(n) * 4);
    L.keys = A.add(size_t(F) * size_t(forest::pow2_at_least(n)) * 8);
    L.weights = A.add(size_t(n) * 4);
    L.s = slot_after(A.bytes(), n, 1);
    return L;
}

// one tree of a launch: its training rows (NULL: rows 0 .. n - 1 of X) and their number
struct RegJob {
    const int32_t *rows;
    int64_t n;
};

}  // namespace

// One CTA per tree of the launch: build_regression_tree with the block as its team.  Tree i's scratch (its weights
// included) starts at scratch + i * L.s.bytes.
__global__ void __launch_bounds__(forest::kThreads) forest_reg_build_kernel(const float *__restrict__ X,
                                                                           const double *__restrict__ y, int F,
                                                                           const RegJob *__restrict__ jobs,
                                                                           const uint32_t *__restrict__ seeds,
                                                                           char *__restrict__ scratch, RegLayout L)
{
    extern __shared__ __align__(16) unsigned char forest_reg_smem[];
    const forest::Team tm{int(threadIdx.x), int(blockDim.x)};
    char *base = scratch + size_t(blockIdx.x) * L.s.bytes;
    const RegJob job = jobs[blockIdx.x];
    forest::RegTree T{X, y, job.rows, reinterpret_cast<const int32_t *>(base + L.weights), job.n, F,
                      reinterpret_cast<int32_t *>(base + L.samples), reinterpret_cast<int32_t *>(base + L.idx),
                      reinterpret_cast<float *>(base + L.fv), reinterpret_cast<uint64_t *>(base + L.keys),
                      reinterpret_cast<forest::StackRec *>(base + L.s.stack), reinterpret_cast<forest::NodeOut *>(base + L.s.nodes),
                      reinterpret_cast<double *>(base + L.s.values)};
    forest::carve_reg_smem(forest_reg_smem, T);
    forest::build_regression_tree(T, tm, seeds[blockIdx.x]);
    put_meta(base + L.s.meta, T.st);
}

extern "C" int b200aa_forest_regressor_fit(const void *d_X, int dtype, int64_t n, int n_feats, int64_t row_stride,
                                           const double *h_y, int n_trees, const int32_t *h_weights,
                                           const uint32_t *h_seeds, b200aa_forest_node *h_nodes, double *h_values,
                                           int64_t node_capacity, int64_t *h_node_count, int32_t *h_max_depth,
                                           void *stream)
{
    NvtxRange nvtx_("b200aa_forest_regressor_fit");
    REFUSE_CAPTURE(stream, "b200aa_forest_regressor_fit", kWhyHostArrays);
    if (!d_X || !h_y || !h_weights || !h_seeds || !h_nodes || !h_values || !h_node_count || !h_max_depth || n < 1 ||
        n > (int64_t(1) << 29) || n_feats < 1 || row_stride < n_feats || n_trees < 1 || node_capacity < 0 ||
        (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (!finite_targets(h_y, n) || !valid_weights(h_weights, int64_t(n_trees) * n)) return B200AA_ERR_INVALID;
    if (n_feats > forest::kMaxFeats) return B200AA_ERR_UNSUPPORTED;
    const RegLayout L = reg_layout(n, n_feats);
    Layout A;
    const size_t x_at = A.add(size_t(n) * n_feats * 4), y_at = A.add(size_t(n) * 8), seeds_at = A.add(size_t(n_trees) * 4),
                 jobs_at = A.add(size_t(n_trees) * sizeof(RegJob));
    const int64_t slice = trees_per_launch(A.bytes(), L.s.bytes, n_trees);
    if (slice < 1) return B200AA_ERR_UNSUPPORTED;
    const size_t trees_at = A.add(size_t(slice) * L.s.bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = forest::reg_smem_bytes(n_feats);
    CK(cudaFuncSetAttribute(forest_reg_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(forest::kRegSmemCap)));
    StreamScratch scratch(st);
    int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    float *Xf = Layout::at<float>(base, x_at);
    double *y = Layout::at<double>(base, y_at);
    uint32_t *seeds = Layout::at<uint32_t>(base, seeds_at);
    RegJob *jobs = Layout::at<RegJob>(base, jobs_at);
    char *trees = Layout::at<char>(base, trees_at);
    if ((rc = cast_to_f32(d_X, dtype, n, n_feats, row_stride, Xf, st)) != B200AA_OK) return rc;
    std::vector<RegJob> hjobs(size_t(slice), RegJob{nullptr, n});
    CK(cudaMemcpyAsync(y, h_y, size_t(n) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(seeds, h_seeds, size_t(n_trees) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(jobs, hjobs.data(), size_t(slice) * sizeof(RegJob), cudaMemcpyHostToDevice, st));
    TreesOut out{h_nodes, h_values, 1, node_capacity, h_node_count, h_max_depth, 0};
    for (int64_t t0 = 0; t0 < n_trees; t0 += slice) {
        const int64_t nt = std::min<int64_t>(slice, n_trees - t0);
        for (int64_t i = 0; i < nt; ++i)
            CK(cudaMemcpyAsync(trees + size_t(i) * L.s.bytes + L.weights, h_weights + (t0 + i) * n, size_t(n) * 4,
                               cudaMemcpyHostToDevice, st));
        forest_reg_build_kernel<<<unsigned(nt), forest::kThreads, smem, st>>>(Xf, y, n_feats, jobs, seeds + t0, trees, L);
        CK_LAUNCH("forest_reg_build_kernel");
        if ((rc = read_trees(st, trees, L.s, t0, nt, out)) != B200AA_OK) return scratch.done(rc);
    }
    return scratch.done(B200AA_OK);
}

// StandardScaler().fit_transform of the whole C-contiguous float64 matrix (kernel 11's front::scaler_fit, rows added in
// sequence), cast to float32 as fit and predict cast it: one thread per column.
__global__ void forest_reg_scale_kernel(const double *__restrict__ X, int64_t n, int F, float *__restrict__ Xs)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    bool inf = false;
    const knn::Scale sc = front::scaler_fit([&](int64_t i) { return X[i * F + f]; }, n, false, inf);
    for (int64_t i = 0; i < n; ++i) Xs[i * F + f] = __double2float_rn(knn::standardise(X[i * F + f], sc));
}

namespace {
// the prediction of one problem's rows by the trees of one launch: problem p's trees are the launch's trees t0 .. t0+nt-1
struct RegPredJob {
    const int32_t *rows;        // the problem's test rows, then its training rows (device)
    int64_t n_rows, acc_off;    // acc_off: the rows' offset in acc and out
    int32_t t0, nt, first, last, n_trees;
};
}  // namespace

// One thread per (problem, row), blockIdx.y the problem: walk its trees of this launch in tree order (forest::tree_apply)
// and add their leaf values to the row's sum (ForestRegressor.predict: out += tree.predict(X)); after the
// problem's last tree, the sum / n_trees in its place (y_hat /= len(estimators_)).
__global__ void forest_reg_predict_kernel(const float *__restrict__ Xs, int F, const RegPredJob *__restrict__ pjobs,
                                          const char *__restrict__ trees, Slot S, double *__restrict__ acc)
{
    const RegPredJob J = pjobs[blockIdx.y];
    const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= J.n_rows) return;
    const float *x = Xs + int64_t(J.rows[r]) * F;
    double a = J.first ? 0.0 : acc[J.acc_off + r];
    for (int t = J.t0; t < J.t0 + J.nt; ++t) {
        const forest::NodeOut *nodes = reinterpret_cast<const forest::NodeOut *>(trees + size_t(t) * S.bytes + S.nodes);
        const double *values = reinterpret_cast<const double *>(trees + size_t(t) * S.bytes + S.values);
        a = forest::dadd(a, values[forest::tree_apply(nodes, [x](int f) { return x[f]; })]);
    }
    acc[J.acc_off + r] = J.last ? forest::ddiv(a, double(J.n_trees)) : a;
}

extern "C" int b200aa_forest_regression_cross_validate(const double *d_X, int64_t n, int n_feats, const double *h_y,
                                                       int64_t n_problems, const int64_t *h_train_off,
                                                       const int32_t *h_train_idx, const int64_t *h_test_off,
                                                       const int32_t *h_test_idx, const int32_t *h_n_trees,
                                                       const int32_t *h_weights, const uint32_t *h_seeds,
                                                       double *d_pred_test, double *d_pred_train, void *stream)
{
    NvtxRange nvtx_("b200aa_forest_regression_cross_validate");
    REFUSE_CAPTURE(stream, "b200aa_forest_regression_cross_validate", kWhyHostArrays);
    if (!d_X || !h_y || !h_train_off || !h_train_idx || !h_test_off || !h_test_idx || !h_n_trees || !h_weights ||
        !h_seeds || !d_pred_test || !d_pred_train || n < 1 || n > (int64_t(1) << 29) || n_feats < 1 || n_problems < 1)
        return B200AA_ERR_INVALID;
    if (!finite_targets(h_y, n) || !valid_splits(n, n_problems, h_train_off, h_train_idx, h_test_off, h_test_idx))
        return B200AA_ERR_INVALID;
    int64_t ntr_max = 0, trees_total = 0, weights_total = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p];
        if (ntr > n || h_n_trees[p] < 1) return B200AA_ERR_INVALID;
        ntr_max = std::max(ntr_max, ntr);
        trees_total += h_n_trees[p];
        weights_total += int64_t(h_n_trees[p]) * ntr;
    }
    if (!valid_weights(h_weights, weights_total)) return B200AA_ERR_INVALID;
    if (n_feats > forest::kMaxFeats) return B200AA_ERR_UNSUPPORTED;
    const int F = n_feats;
    const int64_t n_tr = h_train_off[n_problems], n_te = h_test_off[n_problems], n_rows = n_tr + n_te;
    const RegLayout L = reg_layout(ntr_max, F);
    Layout A;
    const size_t xs_at = A.add(size_t(n) * F * 4), y_at = A.add(size_t(n) * 8), train_at = A.add(size_t(n_tr) * 4),
                 rows_at = A.add(size_t(n_rows) * 4), acc_at = A.add(size_t(std::max<int64_t>(n_rows, 1)) * 8),
                 seeds_at = A.add(size_t(trees_total) * 4), jobs_at = A.add(size_t(trees_total) * sizeof(RegJob)),
                 pjobs_at = A.add(size_t(n_problems) * sizeof(RegPredJob));
    const int64_t slice = std::min<int64_t>(trees_per_launch(A.bytes(), L.s.bytes, trees_total), 65535);    // problems per launch: grid y
    if (slice < 1) return B200AA_ERR_UNSUPPORTED;
    const size_t trees_at = A.add(size_t(slice) * L.s.bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = forest::reg_smem_bytes(F);
    CK(cudaFuncSetAttribute(forest_reg_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(forest::kRegSmemCap)));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    float *d_xs = Layout::at<float>(base, xs_at);
    double *d_y = Layout::at<double>(base, y_at);
    int32_t *d_train = Layout::at<int32_t>(base, train_at), *d_rows = Layout::at<int32_t>(base, rows_at);
    double *d_acc = Layout::at<double>(base, acc_at);
    uint32_t *d_seeds = Layout::at<uint32_t>(base, seeds_at);
    RegJob *d_jobs = Layout::at<RegJob>(base, jobs_at);
    RegPredJob *d_pjobs = Layout::at<RegPredJob>(base, pjobs_at);
    char *d_trees = Layout::at<char>(base, trees_at);
    // every tree's job, and every problem's rows: its test rows, then its training rows
    std::vector<RegJob> jobs(static_cast<size_t>(trees_total));
    std::vector<int32_t> rows(size_t(std::max<int64_t>(n_rows, 1)));
    std::vector<int64_t> tree0(size_t(n_problems) + 1, 0), w0(size_t(n_problems) + 1, 0), row0(size_t(n_problems) + 1, 0);
    std::vector<int32_t> prob_of(static_cast<size_t>(trees_total));
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off[p + 1] - h_test_off[p];
        for (int32_t t = 0; t < h_n_trees[p]; ++t) {
            jobs[size_t(tree0[p] + t)] = RegJob{d_train + h_train_off[p], ntr};
            prob_of[size_t(tree0[p] + t)] = int32_t(p);
        }
        std::copy(h_test_idx + h_test_off[p], h_test_idx + h_test_off[p + 1], rows.begin() + row0[p]);
        std::copy(h_train_idx + h_train_off[p], h_train_idx + h_train_off[p + 1], rows.begin() + row0[p] + nte);
        tree0[p + 1] = tree0[p] + h_n_trees[p];
        w0[p + 1] = w0[p] + int64_t(h_n_trees[p]) * ntr;
        row0[p + 1] = row0[p] + nte + ntr;
    }
    CK(cudaMemcpyAsync(d_y, h_y, size_t(n) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_train, h_train_idx, size_t(n_tr) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_rows, rows.data(), size_t(n_rows) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_seeds, h_seeds, size_t(trees_total) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_jobs, jobs.data(), size_t(trees_total) * sizeof(RegJob), cudaMemcpyHostToDevice, st));
    forest_reg_scale_kernel<<<unsigned((F + 63) / 64), 64, 0, st>>>(d_X, n, F, d_xs);
    CK_LAUNCH("forest_reg_scale_kernel");
    // launches of up to `slice` consecutive trees over the problems' trees in order; after each, every problem with trees
    // in it adds their predictions, in tree order
    std::vector<RegPredJob> pj(static_cast<size_t>(n_problems));
    for (int64_t g0 = 0; g0 < trees_total; g0 += slice) {
        const int64_t nt = std::min<int64_t>(slice, trees_total - g0);
        for (int64_t i = 0; i < nt; ++i) {
            const int64_t g = g0 + i, p = prob_of[size_t(g)];
            const int64_t ntr = h_train_off[p + 1] - h_train_off[p];
            CK(cudaMemcpyAsync(d_trees + size_t(i) * L.s.bytes + L.weights, h_weights + w0[p] + (g - tree0[p]) * ntr,
                               size_t(ntr) * 4, cudaMemcpyHostToDevice, st));
        }
        forest_reg_build_kernel<<<unsigned(nt), forest::kThreads, smem, st>>>(d_xs, d_y, F, d_jobs + g0, d_seeds + g0,
                                                                            d_trees, L);
        CK_LAUNCH("forest_reg_build_kernel");
        int np = 0;
        int64_t max_rows = 0;
        for (int64_t p = prob_of[size_t(g0)]; p < n_problems && tree0[p] < g0 + nt; ++p) {
            const int64_t a = std::max(tree0[p], g0), b = std::min(tree0[p + 1], g0 + nt);
            const int64_t nr = row0[p + 1] - row0[p];
            pj[size_t(np++)] = RegPredJob{d_rows + row0[p], nr, row0[p], int32_t(a - g0), int32_t(b - a), a == tree0[p],
                                          b == tree0[p + 1], h_n_trees[p]};
            max_rows = std::max(max_rows, nr);
        }
        CK(cudaMemcpyAsync(d_pjobs, pj.data(), size_t(np) * sizeof(RegPredJob), cudaMemcpyHostToDevice, st));
        forest_reg_predict_kernel<<<dim3(unsigned((max_rows + 127) / 128), unsigned(np)), 128, 0, st>>>(
            d_xs, F, d_pjobs, d_trees, L.s, d_acc);
        CK_LAUNCH("forest_reg_predict_kernel");
        CK(cudaStreamSynchronize(st));    // the next launch reuses the scratch and the host job arrays
    }
    // every problem's rows: test rows to d_pred_test, training rows to d_pred_train, from the final sums' quotients
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t nte = h_test_off[p + 1] - h_test_off[p], ntr = h_train_off[p + 1] - h_train_off[p];
        if (nte) CK(cudaMemcpyAsync(d_pred_test + h_test_off[p], d_acc + row0[p], size_t(nte) * 8, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(d_pred_train + h_train_off[p], d_acc + row0[p] + nte, size_t(ntr) * 8, cudaMemcpyDeviceToDevice, st));
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernel 13, gradient boosting: one stage of GradientBoostingClassifier fit for many problems (csrc/forest.cuh,
// build_regression_tree with max_depth 3 and boost_leaves), the test rows' raw scores, and the final class counts
// ------------------------------------------------------------------------------------------------
namespace {

// one tree of a stage: problem p's training rows, its [n, K] gradient / raw blocks (tree k reads and updates column k),
// its class indices, and its test rows with their [n_test, K] raw block
struct BoostJob {
    const int32_t *rows;
    int64_t n;
    const double *neg_g;
    const int32_t *y;
    double *raw;
    int32_t k, K;
    const int32_t *test_rows;
    int64_t n_test;
    double *raw_test;
};

// a boosting tree's slot: its leaf arrays, then a regression tree's slot
struct BoostLayout {
    size_t leaf_of, leaf_rows;
    RegLayout reg;
};
BoostLayout boost_layout(int64_t n, int F)
{
    Layout A;
    BoostLayout B;
    B.leaf_of = A.add(size_t(n) * 4);
    B.leaf_rows = A.add(size_t(n) * 4);
    B.reg = reg_layout(n, F, A.bytes());
    return B;
}

}  // namespace

// One CTA per tree of the launch: unit weights, build_regression_tree (max_depth 3) on column k of the problem's negative
// gradient, then boost_leaves: the Newton leaf values and the training rows' raw column k.
__global__ void __launch_bounds__(forest::kThreads) boost_build_kernel(const float *__restrict__ X, int F,
                                                                      const BoostJob *__restrict__ jobs,
                                                                      const uint32_t *__restrict__ seeds, double lr,
                                                                      char *__restrict__ scratch, BoostLayout B)
{
    extern __shared__ __align__(16) unsigned char boost_smem[];
    const forest::Team tm{int(threadIdx.x), int(blockDim.x)};
    const RegLayout &L = B.reg;
    char *base = scratch + size_t(blockIdx.x) * L.s.bytes;
    // forest::carve_reg_smem's carve with part [kThreads] after vpos (boost_smem_bytes), written out: calling the carve
    // here swaps two local arrays in the kernel's stack frame, which costs 16 bytes of stack and 4 / 8 bytes of spill
    // stores / loads
    unsigned char *s = boost_smem;
    forest::RegShared *st = reinterpret_cast<forest::RegShared *>(s);
    s += (sizeof(forest::RegShared) + 15) & ~size_t(15);
    double *vproxy = reinterpret_cast<double *>(s);
    s += size_t(F) * 8;
    int64_t *vpos = reinterpret_cast<int64_t *>(s);
    s += size_t(F) * 8;
    int64_t *part = reinterpret_cast<int64_t *>(s);
    s += size_t(forest::kThreads) * 8;
    float *mn = reinterpret_cast<float *>(s);
    float *mx = mn + F;
    int32_t *features = reinterpret_cast<int32_t *>(mx + F);
    int32_t *constf = features + F, *drawn = constf + F, *vis = drawn + F, *tied = vis + F;
    const BoostJob J = jobs[blockIdx.x];
    int32_t *w = reinterpret_cast<int32_t *>(base + L.weights);
    for (int64_t i = threadIdx.x; i < J.n; i += blockDim.x) w[i] = 1;
    __syncthreads();
    const forest::RegTree T{X, J.neg_g + J.k, J.rows, w, J.n, F,
                            reinterpret_cast<int32_t *>(base + L.samples), reinterpret_cast<int32_t *>(base + L.idx),
                            reinterpret_cast<float *>(base + L.fv), reinterpret_cast<uint64_t *>(base + L.keys),
                            reinterpret_cast<forest::StackRec *>(base + L.s.stack), reinterpret_cast<forest::NodeOut *>(base + L.s.nodes),
                            reinterpret_cast<double *>(base + L.s.values), features, constf, drawn, vis, tied, mn, mx, vproxy,
                            vpos, st, J.K, forest::kBoostDepth};
    forest::build_regression_tree(T, tm, seeds[blockIdx.x]);
    forest::boost_leaves(T, forest::BoostTree{J.y, J.k, J.K, J.raw, lr, reinterpret_cast<int32_t *>(base + B.leaf_of),
                                              reinterpret_cast<int32_t *>(base + B.leaf_rows), part}, tm);
    put_meta(base + L.s.meta, T.st);
}

// One thread per (tree, test row), blockIdx.y the tree of the launch: the row's leaf, and raw_test[:, k] += lr * value
// (predict_stages' update; a stage's trees touch different columns, so their order does not matter)
__global__ void boost_test_kernel(const float *__restrict__ X, int F, const BoostJob *__restrict__ jobs, double lr,
                                  const char *__restrict__ scratch, BoostLayout B)
{
    const BoostJob J = jobs[blockIdx.y];
    const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= J.n_test) return;
    const char *base = scratch + size_t(blockIdx.y) * B.reg.s.bytes;
    const forest::NodeOut *nodes = reinterpret_cast<const forest::NodeOut *>(base + B.reg.s.nodes);
    const double *values = reinterpret_cast<const double *>(base + B.reg.s.values);
    const float *x = X + int64_t(J.test_rows[r]) * F;
    const int32_t leaf = forest::tree_apply(nodes, [x](int f) { return x[f]; });
    double &o = J.raw_test[r * J.K + J.k];
    o = forest::dadd(o, forest::dmul(lr, values[leaf]));
}

namespace {
bool valid_trees_per_stage(int32_t K) { return K == 1 || (K >= 3 && K <= forest::kMaxClasses); }
}  // namespace

extern "C" int b200aa_boosting_stage(const float *d_X, int64_t n_rows, int n_feats, int64_t n_problems,
                                     const int64_t *h_train_off, const int32_t *h_train_rows, const int64_t *h_test_off,
                                     const int32_t *h_test_rows, const int32_t *h_n_trees, const int32_t *h_active,
                                     const int32_t *d_y, const double *d_neg_grad, double *d_raw_train, double *d_raw_test,
                                     const uint32_t *h_seeds, double learning_rate, b200aa_forest_node *h_nodes,
                                     double *h_values, int64_t node_capacity, int64_t *h_node_count, int32_t *h_max_depth,
                                     void *stream)
{
    NvtxRange nvtx_("b200aa_boosting_stage");
    REFUSE_CAPTURE(stream, "b200aa_boosting_stage", kWhyHostArrays);
    const bool out = h_nodes != nullptr;
    if (!d_X || !h_train_off || !h_train_rows || !h_n_trees || !h_active || !d_y || !d_neg_grad || !d_raw_train ||
        !h_seeds || n_rows < 1 || n_rows > (int64_t(1) << 29) || n_feats < 1 || n_problems < 1 ||
        !(learning_rate - learning_rate == 0.0) || (h_test_off == nullptr) != (h_test_rows == nullptr) ||
        out != (h_values != nullptr) || out != (h_node_count != nullptr) || out != (h_max_depth != nullptr) ||
        node_capacity < 0 || !valid_splits(n_rows, n_problems, h_train_off, h_train_rows, h_test_off, h_test_rows))
        return B200AA_ERR_INVALID;
    int64_t ntr_max = 0, nte_max = 0, n_trees = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off ? h_test_off[p + 1] - h_test_off[p] : 0;
        if (!valid_trees_per_stage(h_n_trees[p]) || (h_active[p] != 0 && h_active[p] != 1) || (nte > 0 && !d_raw_test))
            return B200AA_ERR_INVALID;
        if (!h_active[p]) continue;
        ntr_max = std::max(ntr_max, ntr);
        nte_max = std::max(nte_max, nte);
        n_trees += h_n_trees[p];
    }
    if (n_feats > forest::kMaxFeats) return B200AA_ERR_UNSUPPORTED;
    const int64_t n_tr = h_train_off[n_problems], n_te = h_test_off ? h_test_off[n_problems] : 0;
    const BoostLayout B = boost_layout(std::max<int64_t>(ntr_max, 1), n_feats);
    const int64_t n_trees1 = std::max<int64_t>(n_trees, 1);
    Layout A;
    const size_t tr_at = A.add(size_t(n_tr) * 4), te_at = A.add(size_t(std::max<int64_t>(n_te, 1)) * 4),
                 seeds_at = A.add(size_t(n_trees1) * 4), jobs_at = A.add(size_t(n_trees1) * sizeof(BoostJob));
    const int64_t slice = std::min<int64_t>(trees_per_launch(A.bytes(), B.reg.s.bytes, n_trees1), 65535);    // grid y
    if (slice < 1) return B200AA_ERR_UNSUPPORTED;
    if (n_trees == 0) return B200AA_OK;
    const size_t trees_at = A.add(size_t(slice) * B.reg.s.bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = forest::boost_smem_bytes(n_feats);
    CK(cudaFuncSetAttribute(boost_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(forest::kBoostSmemCap)));
    StreamScratch scratch(st);
    int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    int32_t *d_tr = Layout::at<int32_t>(base, tr_at), *d_te = Layout::at<int32_t>(base, te_at);
    uint32_t *d_seeds = Layout::at<uint32_t>(base, seeds_at);
    BoostJob *d_jobs = Layout::at<BoostJob>(base, jobs_at);
    char *d_trees = Layout::at<char>(base, trees_at);
    // every active problem's trees, k inner
    std::vector<BoostJob> jobs;
    jobs.reserve(size_t(n_trees));
    int64_t g_off = 0, t_off = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off ? h_test_off[p + 1] - h_test_off[p] : 0;
        const int32_t K = h_n_trees[p];
        if (h_active[p])
            for (int32_t k = 0; k < K; ++k)
                jobs.push_back(BoostJob{d_tr + h_train_off[p], ntr, d_neg_grad + g_off, d_y + h_train_off[p], d_raw_train + g_off,
                                        k, K, nte ? d_te + h_test_off[p] : nullptr, nte, nte ? d_raw_test + t_off : nullptr});
        g_off += ntr * K;
        t_off += nte * K;
    }
    CK(cudaMemcpyAsync(d_tr, h_train_rows, size_t(n_tr) * 4, cudaMemcpyHostToDevice, st));
    if (n_te) CK(cudaMemcpyAsync(d_te, h_test_rows, size_t(n_te) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_seeds, h_seeds, size_t(n_trees) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_jobs, jobs.data(), size_t(n_trees) * sizeof(BoostJob), cudaMemcpyHostToDevice, st));
    TreesOut trees_out{h_nodes, h_values, 1, node_capacity, h_node_count, h_max_depth, 0};
    for (int64_t t0 = 0; t0 < n_trees; t0 += slice) {
        const int64_t nt = std::min<int64_t>(slice, n_trees - t0);
        boost_build_kernel<<<unsigned(nt), forest::kThreads, smem, st>>>(d_X, n_feats, d_jobs + t0, d_seeds + t0,
                                                                         learning_rate, d_trees, B);
        CK_LAUNCH("boost_build_kernel");
        int64_t te_max = 0;
        for (int64_t i = t0; i < t0 + nt; ++i) te_max = std::max(te_max, jobs[size_t(i)].n_test);
        if (te_max) {
            boost_test_kernel<<<dim3(unsigned((te_max + 127) / 128), unsigned(nt)), 128, 0, st>>>(d_X, n_feats, d_jobs + t0,
                                                                                                learning_rate, d_trees, B);
            CK_LAUNCH("boost_test_kernel");
        }
        // without trees to return, the next launch reuses the scratch in stream order
        if (out && (rc = read_trees(st, d_trees, B.reg.s, t0, nt, trees_out)) != B200AA_OK) return scratch.done(rc);
    }
    return scratch.done(B200AA_OK);
}

extern "C" int b200aa_boosting_scale(const double *d_X, int64_t n, int n_feats, int64_t n_problems,
                                     const int64_t *h_train_off, const int32_t *h_train_idx, const int64_t *h_test_off,
                                     const int32_t *h_test_idx, float *d_Xs, void *stream)
{
    NvtxRange nvtx_("b200aa_boosting_scale");
    REFUSE_CAPTURE(stream, "b200aa_boosting_scale", kWhyHostArrays);
    if (!d_X || !h_train_off || !h_train_idx || !h_test_off || !h_test_idx || !d_Xs || n < 1 || n > (int64_t(1) << 29) ||
        n_feats < 1 || n_problems < 1 || !valid_splits(n, n_problems, h_train_off, h_train_idx, h_test_off, h_test_idx))
        return B200AA_ERR_INVALID;
    const int64_t n_tr = h_train_off[n_problems], n_te = h_test_off[n_problems];
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Layout A;
    const size_t tr_at = A.add(size_t(n_tr) * 4), te_at = A.add(size_t(std::max<int64_t>(n_te, 1)) * 4);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    int32_t *d_tr = Layout::at<int32_t>(scratch.get(), tr_at), *d_te = Layout::at<int32_t>(scratch.get(), te_at);
    CK(cudaMemcpyAsync(d_tr, h_train_idx, size_t(n_tr) * 4, cudaMemcpyHostToDevice, st));
    if (n_te) CK(cudaMemcpyAsync(d_te, h_test_idx, size_t(n_te) * 4, cudaMemcpyHostToDevice, st));
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t ntr = h_train_off[p + 1] - h_train_off[p], nte = h_test_off[p + 1] - h_test_off[p];
        forest_cv_scale_kernel<<<unsigned((n_feats + 63) / 64), 64, 0, st>>>(
            d_X, n_feats, d_tr + h_train_off[p], ntr, d_te + h_test_off[p], nte, d_Xs + h_train_off[p] * n_feats,
            d_Xs + (n_tr + h_test_off[p]) * n_feats);
        CK_LAUNCH("forest_cv_scale_kernel");
    }
    return scratch.done(B200AA_OK);
}

// One thread per test row: predict's class from the row's K raw scores (boost_class), mapped through the problem's present
// classes, and counted as counts[p, y_test, y_pred].
__global__ void boost_count_kernel(const double *__restrict__ raw_test, int64_t n_test, const int32_t *__restrict__ prob,
                                   const int64_t *__restrict__ raw_off, const int64_t *__restrict__ test_off,
                                   const int32_t *__restrict__ trees, const int32_t *__restrict__ classes,
                                   const int32_t *__restrict__ y_test, int n_classes, int32_t *__restrict__ pred,
                                   unsigned long long *__restrict__ counts)
{
    const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= n_test) return;
    const int32_t p = prob[r], K = trees[p];
    const int c = forest::boost_class(raw_test + raw_off[p] + (r - test_off[p]) * K, K);
    const int32_t g = classes[int64_t(p) * forest::kMaxClasses + c];
    pred[r] = g;
    atomicAdd(&counts[(int64_t(p) * n_classes + y_test[r]) * n_classes + g], 1ull);
}

extern "C" int b200aa_boosting_count(const double *d_raw_test, int64_t n_problems, const int64_t *h_test_off,
                                     const int32_t *h_n_trees, const int32_t *h_classes, const int32_t *h_y_test,
                                     int n_classes, int32_t *d_pred, int64_t *d_counts, void *stream)
{
    NvtxRange nvtx_("b200aa_boosting_count");
    REFUSE_CAPTURE(stream, "b200aa_boosting_count", kWhyHostArrays);
    if (!d_raw_test || !h_test_off || !h_n_trees || !h_classes || !h_y_test || !d_pred || !d_counts || n_problems < 1 ||
        n_classes < 2 || n_classes > forest::kMaxClasses || h_test_off[0] != 0)
        return B200AA_ERR_INVALID;
    std::vector<int64_t> raw_off(static_cast<size_t>(n_problems));
    int64_t o = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int32_t K = h_n_trees[p];
        if (!valid_trees_per_stage(K) || h_test_off[p + 1] < h_test_off[p]) return B200AA_ERR_INVALID;
        for (int c = 0; c < (K == 1 ? 2 : K); ++c)
            if (h_classes[p * forest::kMaxClasses + c] < 0 || h_classes[p * forest::kMaxClasses + c] >= n_classes)
                return B200AA_ERR_INVALID;
        for (int64_t i = h_test_off[p]; i < h_test_off[p + 1]; ++i)
            if (h_y_test[i] < 0 || h_y_test[i] >= n_classes) return B200AA_ERR_INVALID;
        raw_off[size_t(p)] = o;
        o += (h_test_off[p + 1] - h_test_off[p]) * K;
    }
    const int64_t n_te = h_test_off[n_problems];
    std::vector<int32_t> prob(size_t(std::max<int64_t>(n_te, 1)));
    for (int64_t p = 0; p < n_problems; ++p)
        for (int64_t i = h_test_off[p]; i < h_test_off[p + 1]; ++i) prob[size_t(i)] = int32_t(p);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CK(cudaMemsetAsync(d_counts, 0, size_t(n_problems) * n_classes * n_classes * sizeof(int64_t), st));
    if (n_te == 0) return B200AA_OK;
    Layout A;
    const size_t prob_at = A.add(size_t(n_te) * 4), off_at = A.add(size_t(n_problems) * 8),
                 toff_at = A.add(size_t(n_problems + 1) * 8), trees_at = A.add(size_t(n_problems) * 4),
                 cls_at = A.add(size_t(n_problems) * forest::kMaxClasses * 4), y_at = A.add(size_t(n_te) * 4);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(A.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    int32_t *d_prob = Layout::at<int32_t>(base, prob_at);
    int64_t *d_off = Layout::at<int64_t>(base, off_at), *d_toff = Layout::at<int64_t>(base, toff_at);
    int32_t *d_trees = Layout::at<int32_t>(base, trees_at), *d_cls = Layout::at<int32_t>(base, cls_at);
    int32_t *d_y = Layout::at<int32_t>(base, y_at);
    CK(cudaMemcpyAsync(d_prob, prob.data(), size_t(n_te) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_off, raw_off.data(), size_t(n_problems) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_toff, h_test_off, size_t(n_problems + 1) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_trees, h_n_trees, size_t(n_problems) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_cls, h_classes, size_t(n_problems) * forest::kMaxClasses * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_y, h_y_test, size_t(n_te) * 4, cudaMemcpyHostToDevice, st));
    boost_count_kernel<<<unsigned((n_te + 127) / 128), 128, 0, st>>>(d_raw_test, n_te, d_prob, d_off, d_toff, d_trees, d_cls,
                                                                     d_y, n_classes, d_pred,
                                                                     reinterpret_cast<unsigned long long *>(d_counts));
    CK_LAUNCH("boost_count_kernel");
    return scratch.done(B200AA_OK);
}
