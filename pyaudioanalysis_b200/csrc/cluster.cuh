// Cluster distance means (kernel 9): the silhouette terms of speaker_diarization (reference audioSegmentation.py:943-985)
// for one clustering of the rows of X [n, D], bit for bit NumPy and scipy:
//
//   A[c]      = np.mean(pdist(X[labels == c].T))          distances between the D columns over cluster c's rows
//   B[c, c2]  = np.mean(cdist(X[labels == c], X[labels == c2]))
//
//   distance  sqrt(((u_0 - v_0)^2 + (u_1 - v_1)^2) + ...), scipy's sequential fp64 chain (knn.cuh's dist_step);
//   mean      np.add.reduce over the row-major flattening of the n_c x n_c2 block, or over pdist's condensed vector, is one
//             pairwise sum (npsum.cuh) over all its elements; then one division by the count.  No terms: NaN.
//
// A mean of N terms is cut into 2^L segments, the subtrees of its pairwise tree at depth L (npy::pairwise_part), each at
// most kSegTerms long; a segment is cut further into 2^levels leaves of at most 128 terms.  A leaf adds its terms as
// NumPy's leaf does (eight running sums, combined, then the tail); the leaf sums of a segment and the segment sums of a
// mean are combined in tree order (combine).  A leaf or segment at or past the end of a shorter branch is empty and adds
// +0.0, which changes no sum of distances (every term is >= +0 or NaN).
//
// The plan (make_plan) is host code shared by the library and tests/cluster_host.cu; the arithmetic pieces are
// __host__ __device__, so the host test runs the kernels' own order of operations.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

#include "knn.cuh"
#include "npsum.cuh"

namespace b200aa {
namespace cluster {

using npy::dadd;
using npy::ddiv;

constexpr int kTile = 64;                       // items per side of a distance tile
constexpr int kF = 16;                          // chain terms staged in shared memory per step
constexpr int kThreads = 256;                   // 16 x 16 threads, each a 4 x 4 register tile of distance chains
constexpr int64_t kSegTerms = int64_t(1) << 22; // terms of one segment at most (32 MiB of distances)
constexpr int64_t kPassTerms = int64_t(1) << 24;// distances computed per pass, unless one segment needs more
constexpr int kMaxFeats = 4096;                 // D: a pdist mean is never split (its one segment holds all D (D - 1) / 2
                                                // terms, 8 386 560 at D = 4096, past kSegTerms) and its pass holds them

enum : int32_t { kBlock = 0, kPdist = 1 };

// One segment: terms [term0, term0 + len) of the distances a pass computes for it from dist0 on.
//   kBlock  left item u is row left0 + u of the gathered matrix G [n, D], right item v row right0 + v; the chain runs over
//           the D features; distance (u, v) lands at dist0 + u * n_right + v.  The left items are the rows of cluster c
//           that the segment's range of the flattened block touches, all n_right = n_c2 rows of c2 on the right.
//   kPdist  item u is column u of the n_feat = n_c rows left0 ..; distance (u, v), u < v, lands at dist0 + its condensed
//           index; n_left = n_right = D.
struct Segment {
    int64_t left0, right0, n_left, n_right, n_feat;
    int64_t dist0, term0, len;
    int64_t tile0, leaf0;                       // first distance tile / leaf of the segment in its pass
    int32_t kind, levels;                       // levels: leaf_levels(len)
};

// pdist's condensed index of (u, v), u < v, among d items
__host__ __device__ inline int64_t condensed(int64_t u, int64_t v, int64_t d) { return u * d - u * (u + 1) / 2 + (v - u - 1); }

// The depth at which every part of pairwise_sum(n)'s tree is at most `cap` (>= kLeaf) long: the right half of a split is
// never the shorter, so the rightmost branch is the deepest.
__host__ __device__ inline int part_levels(int64_t n, int64_t cap)
{
    int d = 0;
    while (n > cap) {
        int64_t n2 = n / 2;
        n2 -= n2 % 8;
        n -= n2;
        ++d;
    }
    return d;
}
__host__ __device__ inline int leaf_levels(int64_t n) { return part_levels(n, npy::kLeaf); }

// NumPy's leaf of n <= 128 terms, as 8 lanes compute it: lane j's running sum over terms j, j + 8, ... below n - n % 8
// (n >= 8; for n < 8 lane 0 holds the sequential sum from 0.0 and the others 0.0) ...
template <class G>
__host__ __device__ double leaf_lane(const G &get, int64_t n, int j)
{
    if (n < 8) {
        double r = 0.0;
        if (j == 0)
            for (int64_t i = 0; i < n; ++i) r = dadd(r, get(i));
        return r;
    }
    double r = get(j);
    for (int64_t i = 8 + j; i < n - (n % 8); i += 8) r = dadd(r, get(i));
    return r;
}
// ... then ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) plus the tail in sequence
template <class G>
__host__ __device__ double leaf_finish(const double *r, const G &get, int64_t n)
{
    if (n < 8) return r[0];
    double res = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
    for (int64_t i = n - (n % 8); i < n; ++i) res = dadd(res, get(i));
    return res;
}

// the 2^levels part sums s[0 ..] of a tree combined in place in tree order, the serial statement of the kernels' passes
__host__ __device__ inline double combine(double *s, int levels)
{
    for (int j = 0; j < levels; ++j)
        for (int64_t k = 0; k + (int64_t(1) << j) < (int64_t(1) << levels); k += int64_t(2) << j)
            s[k] = dadd(s[k], s[k + (int64_t(1) << j)]);
    return s[0];
}

// One mean: its 2^levels segments from seg0 on, its term count, and where it goes in out [K + K * K] (A, then B row-major)
struct Mean {
    int64_t seg0, count;
    int32_t levels, slot;
};

// The work of one clustering: the means asked for, their segments, and the passes that run them.  A pass is the segments
// [pass_seg[p], pass_seg[p + 1]) with pass_dist[p] distances, pass_tiles[p] tiles and pass_leaves[p] leaves.
struct Plan {
    std::vector<Mean> means;
    std::vector<Segment> segs;
    std::vector<int64_t> pass_seg, pass_dist, pass_tiles, pass_leaves;
};

inline int64_t tiles_of(const Segment &s)
{
    return ((s.n_left + kTile - 1) / kTile) * ((s.n_right + kTile - 1) / kTile);
}

// off[0 .. K]: the clusters' first rows in G (rows in cluster order); want[c]: compute A[c] and B[c, *].
inline void make_plan(const int64_t *off, int K, int D, const unsigned char *want, int64_t seg_terms, int64_t pass_terms,
                      Plan &plan)
{
    auto add_mean = [&](int slot, int kind, int c, int c2, int64_t count) {
        Mean m;
        m.seg0 = int64_t(plan.segs.size());
        m.count = count;
        m.levels = kind == kBlock ? part_levels(count, seg_terms) : 0;
        m.slot = slot;
        plan.means.push_back(m);
        const int64_t n2 = kind == kBlock ? off[c2 + 1] - off[c2] : D;
        for (int k = 0; k < (1 << m.levels); ++k) {
            Segment s{};
            int64_t a = 0, len = count;
            npy::pairwise_part(count, m.levels, k, a, len);
            s.kind = kind;
            s.len = len;
            s.levels = leaf_levels(len);
            if (kind == kBlock) {
                const int64_t r0 = len ? a / n2 : 0, r1 = len ? (a + len - 1) / n2 + 1 : 0;
                s.left0 = off[c] + r0;
                s.right0 = off[c2];
                s.n_left = r1 - r0;
                s.n_right = n2;
                s.n_feat = D;
                s.term0 = len ? a - r0 * n2 : 0;
            } else {
                s.left0 = s.right0 = off[c];
                s.n_left = s.n_right = D;
                s.n_feat = off[c + 1] - off[c];
                s.term0 = 0;
            }
            plan.segs.push_back(s);
        }
    };
    for (int c = 0; c < K; ++c) {
        if (!want[c]) continue;
        const int64_t nc = off[c + 1] - off[c];
        if (D >= 2) add_mean(c, kPdist, c, c, int64_t(D) * (D - 1) / 2);
        for (int c2 = 0; c2 < K; ++c2) {
            const int64_t n = nc * (off[c2 + 1] - off[c2]);
            if (c2 != c && n > 0) add_mean(K + c * K + c2, kBlock, c, c2, n);
        }
    }
    plan.pass_seg.assign(1, 0);
    int64_t dist = 0, tiles = 0, leaves = 0;
    for (size_t i = 0; i < plan.segs.size(); ++i) {
        Segment &s = plan.segs[i];
        const int64_t nd = s.kind == kBlock ? s.n_left * s.n_right : int64_t(D) * (D - 1) / 2;
        if (i > size_t(plan.pass_seg.back()) && dist + nd > pass_terms) {
            plan.pass_seg.push_back(int64_t(i));
            plan.pass_dist.push_back(dist);
            plan.pass_tiles.push_back(tiles);
            plan.pass_leaves.push_back(leaves);
            dist = tiles = leaves = 0;
        }
        s.dist0 = dist;
        s.tile0 = tiles;
        s.leaf0 = leaves;
        dist += nd;
        tiles += tiles_of(s);
        leaves += int64_t(1) << s.levels;
    }
    plan.pass_seg.push_back(int64_t(plan.segs.size()));
    plan.pass_dist.push_back(dist);
    plan.pass_tiles.push_back(tiles);
    plan.pass_leaves.push_back(leaves);
}

// the chain term f of items u (left) and v (right) of segment s: G [n, D] row-major
__host__ __device__ inline double left_at(const Segment &s, const double *G, int D, int64_t u, int64_t f)
{
    return s.kind == kBlock ? G[(s.left0 + u) * D + f] : G[(s.left0 + f) * D + u];
}
__host__ __device__ inline double right_at(const Segment &s, const double *G, int D, int64_t v, int64_t f)
{
    return s.kind == kBlock ? G[(s.right0 + v) * D + f] : G[(s.left0 + f) * D + v];
}
// where distance (u, v) lands, or -1 when pdist does not compute it (v <= u)
__host__ __device__ inline int64_t dist_index(const Segment &s, int64_t u, int64_t v)
{
    if (s.kind == kBlock) return s.dist0 + u * s.n_right + v;
    return v > u ? s.dist0 + condensed(u, v, s.n_left) : -1;
}

}  // namespace cluster
}  // namespace b200aa

// The distance tile kernel (cluster.cu): segments [s0, s1) of a pass, G's rows `D` doubles apart.  Kernel 11's outlier rule
// (front.cu) launches it too, on one kBlock segment of every pair of columns.
__global__ void __launch_bounds__(b200aa::cluster::kThreads, 2)
cluster_dist_kernel(const b200aa::cluster::Segment *__restrict__ segs, int64_t s0, int64_t s1, const double *__restrict__ G,
                    int D, double *__restrict__ dist);
