// Host program for tests/test_cluster_cpu.py: runs kernel 9's plan and its __host__ __device__ pieces
// (pyaudioanalysis_b200/csrc/cluster.cuh) on the CPU in the order the kernels apply them.  Reads commands from stdin,
// numbers as C hex floats / "inf" / "nan"; prints hex floats ("nan" for NaN).
//
//   means K D n seg_terms pass_terms labels (n) want (K) X (n x D)  -> A (K) then B (K x K)
//   dist kind n D X (n x D)     kind 0: cdist(X, X) (n x n); kind 1: pdist(X.T) (D (D - 1) / 2)
//   bigsum N seg_terms          a pairwise sum of N generated terms, by segments and leaves, then npy::pairwise_sum;
//                               also checks that the segments tile [0, N) and every leaf holds at most 128 terms
//   plan K D sizes (K)          make_plan at the library's kSegTerms / kPassTerms for every cluster of the given sizes:
//                               seg_terms pass_terms n_passes, then per segment in plan order: kind, mean slot, len, pass
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/cluster.cuh"
#include "host_io.h"

using namespace b200aa;

// the distance of items u, v of segment s: the kernel's chain
static double chain(const cluster::Segment &s, const double *G, int D, int64_t u, int64_t v)
{
    double acc = 0.0;
    for (int64_t f = 0; f < s.n_feat; ++f) acc = knn::dist_step(acc, cluster::left_at(s, G, D, u, f), cluster::right_at(s, G, D, v, f));
    return npy::dsqrt(acc);
}

// the 8-lane leaf of cluster_leaf_kernel
template <class Get>
static double leaf(const Get &get, int64_t len)
{
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = cluster::leaf_lane(get, len, j);
    return cluster::leaf_finish(r, get, len);
}

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "means")) {
            const int K = int(rl()), D = int(rl());
            const int64_t n = rl(), seg_terms = rl(), pass_terms = rl();
            std::vector<int> labels(n);
            for (auto &l : labels) l = int(rl());
            std::vector<unsigned char> want(K);
            for (auto &w : want) w = (unsigned char)rl();
            const std::vector<double> X = rv(size_t(n) * D);
            // G: the rows of each cluster together, in ascending order (cluster_gather_kernel)
            std::vector<int64_t> off(K + 1, 0);
            for (int l : labels) ++off[l + 1];
            for (int c = 0; c < K; ++c) off[c + 1] += off[c];
            std::vector<int64_t> fill(off.begin(), off.end() - 1);
            std::vector<double> G(X.size());
            for (int64_t i = 0; i < n; ++i) {
                const int64_t r = fill[labels[i]]++;
                for (int f = 0; f < D; ++f) G[size_t(r) * D + f] = X[size_t(i) * D + f];
            }
            cluster::Plan plan;
            cluster::make_plan(off.data(), K, D, want.data(), seg_terms, pass_terms, plan);
            std::vector<double> seg_sum(plan.segs.size());
            for (size_t p = 0; p + 1 < plan.pass_seg.size(); ++p) {
                if (plan.pass_dist[p] > pass_terms && plan.pass_seg[p + 1] - plan.pass_seg[p] > 1) return 3;
                std::vector<double> dist(size_t(plan.pass_dist[p]), -1.0), leaf_sum(size_t(plan.pass_leaves[p]));
                for (int64_t g = plan.pass_seg[p]; g < plan.pass_seg[p + 1]; ++g) {          // cluster_dist_kernel
                    const cluster::Segment &s = plan.segs[g];
                    for (int64_t u = 0; u < s.n_left; ++u)
                        for (int64_t v = 0; v < s.n_right; ++v) {
                            const int64_t at = cluster::dist_index(s, u, v);
                            if (at >= 0) dist[size_t(at)] = chain(s, G.data(), D, u, v);
                        }
                }
                for (int64_t g = plan.pass_seg[p]; g < plan.pass_seg[p + 1]; ++g) {          // leaf and combine kernels
                    const cluster::Segment &s = plan.segs[g];
                    for (int k = 0; k < (1 << s.levels); ++k) {
                        int64_t o = 0, len = 0;
                        npy::pairwise_part(s.len, s.levels, k, o, len);
                        if (len > npy::kLeaf) return 4;
                        const double *d = dist.data() + s.dist0 + s.term0 + o;
                        leaf_sum[size_t(s.leaf0 + k)] = leaf([d](int64_t i) { return d[i]; }, len);
                    }
                    seg_sum[size_t(g)] = cluster::combine(leaf_sum.data() + s.leaf0, s.levels);
                }
            }
            std::vector<double> out(size_t(K) + size_t(K) * K, NAN);                           // cluster_mean_kernel
            for (const cluster::Mean &m : plan.means)
                out[size_t(m.slot)] = npy::ddiv(cluster::combine(seg_sum.data() + m.seg0, m.levels), double(m.count));
            printf("means");
            for (double v : out) pr(v);
            printf("\n");
        } else if (!strcmp(cmd, "dist")) {
            const int kind = int(rl());
            const int64_t n = rl();
            const int D = int(rl());
            const std::vector<double> X = rv(size_t(n) * D);
            cluster::Segment s{};
            s.kind = kind;
            if (kind == cluster::kBlock) {
                s.n_left = s.n_right = n;
                s.n_feat = D;
            } else {
                s.n_left = s.n_right = D;
                s.n_feat = n;
            }
            std::vector<double> dist(kind == cluster::kBlock ? size_t(n) * n : size_t(D) * (D - 1) / 2);
            for (int64_t u = 0; u < s.n_left; ++u)
                for (int64_t v = 0; v < s.n_right; ++v) {
                    const int64_t at = cluster::dist_index(s, u, v);
                    if (at >= 0) dist[size_t(at)] = chain(s, X.data(), D, u, v);
                }
            printf("dist");
            for (double v : dist) pr(v);
            printf("\n");
        } else if (!strcmp(cmd, "bigsum")) {
            const int64_t N = rl(), seg_terms = rl();
            // terms >= +0 spread over many binades: the sum depends on the order of the additions
            auto term = [](int64_t i) {
                uint64_t h = uint64_t(i) * 0x9E3779B97F4A7C15ull;
                h ^= h >> 29;
                h *= 0xBF58476D1CE4E5B9ull;
                h ^= h >> 32;
                return std::ldexp(double(h >> 11), int(h & 31) - 53);
            };
            const int L = cluster::part_levels(N, seg_terms);
            std::vector<double> seg(size_t(1) << L);
            int64_t next = 0;
            for (int k = 0; k < (1 << L); ++k) {
                int64_t a = 0, len = 0;
                npy::pairwise_part(N, L, k, a, len);
                if (len > seg_terms || (len && a != next)) return 5;
                next += len;
                const int lv = cluster::leaf_levels(len);
                std::vector<double> leaves(size_t(1) << lv);
                for (int j = 0; j < (1 << lv); ++j) {
                    int64_t o = 0, ll = 0;
                    npy::pairwise_part(len, lv, j, o, ll);
                    if (ll > npy::kLeaf) return 4;
                    leaves[size_t(j)] = leaf([&](int64_t i) { return term(a + o + i); }, ll);
                }
                seg[size_t(k)] = cluster::combine(leaves.data(), lv);
            }
            if (next != N) return 5;
            printf("bigsum");
            pr(cluster::combine(seg.data(), L));
            pr(npy::pairwise_sum(term, 0, N, N));
            printf("\n");
        } else if (!strcmp(cmd, "plan")) {
            const int K = int(rl()), D = int(rl());
            std::vector<int64_t> off(K + 1, 0);
            for (int c = 0; c < K; ++c) off[c + 1] = off[c] + rl();
            const std::vector<unsigned char> want(K, 1);
            cluster::Plan plan;
            cluster::make_plan(off.data(), K, D, want.data(), cluster::kSegTerms, cluster::kPassTerms, plan);
            std::vector<int> slot(plan.segs.size()), pass(plan.segs.size());
            for (const cluster::Mean &m : plan.means)
                for (int k = 0; k < (1 << m.levels); ++k) slot[size_t(m.seg0 + k)] = m.slot;
            for (size_t p = 0; p + 1 < plan.pass_seg.size(); ++p)
                for (int64_t g = plan.pass_seg[p]; g < plan.pass_seg[p + 1]; ++g) pass[size_t(g)] = int(p);
            printf("plan %lld %lld %d", (long long)cluster::kSegTerms, (long long)cluster::kPassTerms,
                   int(plan.pass_seg.size()) - 1);
            for (size_t g = 0; g < plan.segs.size(); ++g)
                printf(" %d %d %lld %d", plan.segs[g].kind, slot[g], (long long)plan.segs[g].len, pass[g]);
            printf("\n");
        } else {
            return 2;
        }
    }
    return 0;
}
