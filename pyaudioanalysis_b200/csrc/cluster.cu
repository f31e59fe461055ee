// libb200aa.so -- cluster distance means (kernel 9).
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/b200aa.h"
#include "cluster.cuh"
#include "entry.h"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 9: the silhouette means of speaker_diarization (audioSegmentation.py:943-985), bit for bit np.mean of scipy's
// pdist / cdist (csrc/cluster.cuh)
// ------------------------------------------------------------------------------------------------
// G[r] = X[perm[r]]: the rows of every cluster together, each cluster's in ascending row order.
__global__ void __launch_bounds__(256) cluster_gather_kernel(const double *__restrict__ X, int64_t x_stride, int D,
                                                             const int64_t *__restrict__ perm, int64_t n,
                                                             double *__restrict__ G)
{
    for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < n * D; e += int64_t(gridDim.x) * blockDim.x) {
        const int64_t r = e / D, f = e - r * D;
        G[e] = X[perm[r] * x_stride + f];
    }
}

// the segment of [s0, s1) whose first entry (tile0 or leaf0) is the last at or below i: the one that owns i
template <class Key>
__device__ inline int64_t owner(const cluster::Segment *__restrict__ segs, int64_t s0, int64_t s1, int64_t i, Key key)
{
    int64_t lo = s0, hi = s1;                   // first segment whose key is above i, by bisection
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        if (key(segs[mid]) <= i) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// One 64 x 64 tile of a segment's distances per CTA.  Both sides are staged kF chain terms at a time, as [term][item];
// each thread runs 4 x 4 independent chains (left items ty + 16a, right items tx + 16b), as knn_dist_kernel does.
__global__ void __launch_bounds__(cluster::kThreads, 2) cluster_dist_kernel(const cluster::Segment *__restrict__ segs,
                                                                         int64_t s0, int64_t s1,
                                                                         const double *__restrict__ G, int D,
                                                                         double *__restrict__ dist)
{
    using namespace cluster;
    __shared__ double sl[kF][kTile + 1];
    __shared__ double sr[kF][kTile + 1];
    const int64_t t = blockIdx.x;
    const Segment s = segs[owner(segs, s0, s1, t, [](const Segment &g) { return g.tile0; })];
    const int64_t lt = t - s.tile0, tiles_v = (s.n_right + kTile - 1) / kTile;
    const int64_t u0 = (lt / tiles_v) * kTile, v0 = (lt % tiles_v) * kTile;
    if (s.kind == kPdist && v0 + kTile - 1 <= u0) return;      // pdist keeps u < v only
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int64_t f0 = 0; f0 < s.n_feat; f0 += kF) {
        const int nf = int(min(int64_t(kF), s.n_feat - f0));
        __syncthreads();
        for (int e = threadIdx.x; e < kTile * kF; e += kThreads) {
            // consecutive threads on consecutive addresses: along the features of a row (kBlock), along a row (kPdist)
            const int r = s.kind == kBlock ? e / kF : e % kTile, j = s.kind == kBlock ? e % kF : e / kTile;
            const int64_t u = u0 + r, v = v0 + r;
            sl[j][r] = (j < nf && u < s.n_left) ? left_at(s, G, D, u, f0 + j) : 0.0;
            sr[j][r] = (j < nf && v < s.n_right) ? right_at(s, G, D, v, f0 + j) : 0.0;
        }
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < nf; ++j) {
            double x[4], y[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) x[a] = sl[j][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 4; ++b) y[b] = sr[j][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = knn::dist_step(acc[a][b], x[a], y[b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int64_t u = u0 + ty + 16 * a;
        if (u >= s.n_left) continue;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int64_t v = v0 + tx + 16 * b;
            const int64_t at = v < s.n_right ? dist_index(s, u, v) : -1;
            if (at >= 0) dist[at] = npy::dsqrt(acc[a][b]);
        }
    }
}

// Eight lanes per leaf: lane j's running sum (cluster::leaf_lane), gathered by shuffles into the group's first lane, which
// finishes the leaf and writes its sum.
__global__ void __launch_bounds__(256) cluster_leaf_kernel(const cluster::Segment *__restrict__ segs, int64_t s0, int64_t s1,
                                                           int64_t n_leaves, const double *__restrict__ dist,
                                                           double *__restrict__ leaf_sum)
{
    using namespace cluster;
    const int64_t leaf = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 3;
    const int j = threadIdx.x & 7;
    const bool live = leaf < n_leaves;
    int64_t off = 0, len = 0;
    const double *d = dist;
    if (live) {
        const Segment s = segs[owner(segs, s0, s1, leaf, [](const Segment &g) { return g.leaf0; })];
        npy::pairwise_part(s.len, s.levels, int(leaf - s.leaf0), off, len);
        d = dist + s.dist0 + s.term0 + off;
    }
    auto get = [d](int64_t i) { return d[i]; };
    double r[8];
    const double mine = live ? leaf_lane(get, len, j) : 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = __shfl_sync(0xffffffffu, mine, (threadIdx.x & 31 & ~7) + k);
    if (live && j == 0) leaf_sum[leaf] = leaf_finish(r, get, len);
}

// One CTA per segment of the pass: its 2^levels leaf sums combined in place in tree order (cluster::combine, one level per
// step), the result stored as the segment's sum.
__global__ void __launch_bounds__(256) cluster_combine_kernel(const cluster::Segment *__restrict__ segs, int64_t s0,
                                                              double *__restrict__ leaf_sum, double *__restrict__ seg_sum)
{
    const int64_t g = s0 + blockIdx.x;
    const cluster::Segment s = segs[g];
    double *v = leaf_sum + s.leaf0;
    const int64_t n = int64_t(1) << s.levels;
    for (int j = 0; j < s.levels; ++j) {
        const int64_t h = int64_t(1) << j;
        for (int64_t k = int64_t(threadIdx.x) * 2 * h; k < n; k += int64_t(blockDim.x) * 2 * h) v[k] = npy::dadd(v[k], v[k + h]);
        __syncthreads();
    }
    if (threadIdx.x == 0) seg_sum[g] = v[0];
}

// One thread per output: its mean's segment sums combined in tree order and divided by the count, or NaN
__global__ void __launch_bounds__(128) cluster_mean_kernel(const cluster::Mean *__restrict__ means,
                                                           const int32_t *__restrict__ mean_of, int K,
                                                           double *__restrict__ seg_sum, double *__restrict__ A,
                                                           double *__restrict__ B)
{
    const int64_t slot = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (slot >= K + int64_t(K) * K) return;
    double v = __longlong_as_double(0x7ff8000000000000ll);
    const int32_t m = mean_of[slot];
    if (m >= 0) {
        const cluster::Mean mn = means[m];
        v = npy::ddiv(cluster::combine(seg_sum + mn.seg0, mn.levels), double(mn.count));
    }
    if (slot < K) A[slot] = v;
    else B[slot - K] = v;
}

extern "C" int b200aa_cluster_distance_means(const double *d_X, int64_t n, int n_feats, int64_t x_stride,
                                             const int32_t *h_labels, int n_clusters, const unsigned char *h_want,
                                             double *d_A, double *d_B, void *stream)
{
    NvtxRange nvtx_("b200aa_cluster_distance_means");
    REFUSE_CAPTURE(stream, "b200aa_cluster_distance_means", kWhyHostArrays);
    const int K = n_clusters, D = n_feats;
    if (!d_X || !h_labels || !d_A || !d_B || n < 1 || D < 1 || D > cluster::kMaxFeats || x_stride < D || K < 1 ||
        K > B200AA_CLUSTER_MAX)
        return B200AA_ERR_INVALID;
    std::vector<int64_t> off(size_t(K) + 1, 0);
    for (int64_t i = 0; i < n; ++i) {
        if (h_labels[i] < 0 || h_labels[i] >= K) return B200AA_ERR_INVALID;
        ++off[size_t(h_labels[i]) + 1];
    }
    for (int c = 0; c < K; ++c) off[c + 1] += off[c];
    std::vector<int64_t> perm(static_cast<size_t>(n)), fill(off.begin(), off.end() - 1);
    for (int64_t i = 0; i < n; ++i) perm[size_t(fill[size_t(h_labels[i])]++)] = i;
    std::vector<unsigned char> want(size_t(K), 1);
    if (h_want) std::copy(h_want, h_want + K, want.begin());
    cluster::Plan plan;
    cluster::make_plan(off.data(), K, D, want.data(), cluster::kSegTerms, cluster::kPassTerms, plan);
    const int64_t n_slots = K + int64_t(K) * K;
    std::vector<int32_t> mean_of(size_t(n_slots), -1);
    for (size_t m = 0; m < plan.means.size(); ++m) mean_of[size_t(plan.means[m].slot)] = int32_t(m);

    // the permutation, segments, means and mean_of, uploaded at once as one head
    Layout L;
    const size_t perm_at = L.add(perm.size() * sizeof(int64_t)), segs_at = L.add(plan.segs.size() * sizeof(cluster::Segment)),
                 means_at = L.add(plan.means.size() * sizeof(cluster::Mean)), mean_of_at = L.add(mean_of.size() * sizeof(int32_t));
    std::vector<char> head(L.bytes(), 0);
    std::memcpy(head.data() + perm_at, perm.data(), perm.size() * sizeof(int64_t));
    std::memcpy(head.data() + segs_at, plan.segs.data(), plan.segs.size() * sizeof(cluster::Segment));
    std::memcpy(head.data() + means_at, plan.means.data(), plan.means.size() * sizeof(cluster::Mean));
    std::memcpy(head.data() + mean_of_at, mean_of.data(), mean_of.size() * sizeof(int32_t));
    // then G, the segment sums, and the largest pass's distances and leaf sums
    const size_t g_at = L.add(size_t(n) * D * sizeof(double)), sums_at = L.add(plan.segs.size() * sizeof(double)),
                 dist_at = L.add(size_t(*std::max_element(plan.pass_dist.begin(), plan.pass_dist.end())) * sizeof(double)),
                 leaf_at = L.add(size_t(*std::max_element(plan.pass_leaves.begin(), plan.pass_leaves.end())) * sizeof(double));

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(L.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const int64_t *d_perm = Layout::at<const int64_t>(base, perm_at);
    const cluster::Segment *d_segs = Layout::at<const cluster::Segment>(base, segs_at);
    const cluster::Mean *d_means = Layout::at<const cluster::Mean>(base, means_at);
    const int32_t *d_mean_of = Layout::at<const int32_t>(base, mean_of_at);
    double *G = Layout::at<double>(base, g_at), *seg_sum = Layout::at<double>(base, sums_at);
    double *dist = Layout::at<double>(base, dist_at), *leaf_sum = Layout::at<double>(base, leaf_at);
    CK(cudaMemcpyAsync(base, head.data(), head.size(), cudaMemcpyHostToDevice, st));
    const int64_t cells = n * D;
    cluster_gather_kernel<<<unsigned(std::min<int64_t>((cells + 255) / 256, 1 << 16)), 256, 0, st>>>(d_X, x_stride, D, d_perm,
                                                                                                     n, G);
    CK_LAUNCH("cluster_gather_kernel");
    for (size_t p = 0; p + 1 < plan.pass_seg.size(); ++p) {
        const int64_t s0 = plan.pass_seg[p], s1 = plan.pass_seg[p + 1];
        if (s0 == s1) continue;
        if (plan.pass_tiles[p]) {
            cluster_dist_kernel<<<unsigned(plan.pass_tiles[p]), cluster::kThreads, 0, st>>>(d_segs, s0, s1, G, D, dist);
            CK_LAUNCH("cluster_dist_kernel");
        }
        cluster_leaf_kernel<<<unsigned((plan.pass_leaves[p] + 31) / 32), 256, 0, st>>>(d_segs, s0, s1, plan.pass_leaves[p], dist,
                                                                                      leaf_sum);
        CK_LAUNCH("cluster_leaf_kernel");
        cluster_combine_kernel<<<unsigned(s1 - s0), 256, 0, st>>>(d_segs, s0, leaf_sum, seg_sum);
        CK_LAUNCH("cluster_combine_kernel");
    }
    cluster_mean_kernel<<<unsigned((n_slots + 127) / 128), 128, 0, st>>>(d_means, d_mean_of, K, seg_sum, d_A, d_B);
    CK_LAUNCH("cluster_mean_kernel");
    return scratch.done(B200AA_OK);
}
