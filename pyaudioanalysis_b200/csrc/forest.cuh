// Forest training (kernel 13): scikit-learn 1.9's RandomForestClassifier / ExtraTreesClassifier fit with the library's
// arguments (all defaults: gini, max_features="sqrt", min_samples_split=2, min_samples_leaf=1, no depth limit), one tree
// node for node, bit for bit.
//
// Why it can be exact: every sample weight is an integer (bootstrap counts, or 1), so every class count and weighted_n_*
// is an exact integer in any summation order; a split candidate lies only between two sorted float32 values more than
// FEATURE_THRESHOLD apart, so the counts at a candidate do not depend on how equal values were ordered, and the partition
// goes by x <= threshold.  What is left is fixed-order float64 arithmetic on those integers (written here with the _rn
// operations of npsum.cuh: no contraction) and the splitter's our_rand_r stream, restated below.
//
// build_tree() is the whole DepthFirstTreeBuilder loop for one tree, written for a team of threads: on the device one
// CTA (Team = the block, sync = __syncthreads), in tests/forest_host.cu a team of one thread on the CPU.  Per node:
//   1. class totals and, for every feature, min / max over the node's samples (team-parallel);
//   2. thread 0 runs node_split_best / node_split_random's Fisher-Yates draw loop with the known / found / drawn
//      constant bookkeeping and the two memcpys (draw_features); the random splitter's thresholds are drawn there too;
//   3. each drawn non-constant feature in visit order: best splitter: the node's (value, sample) keys bitonic-sorted in
//      global scratch, prefix class counts per thread chunk, the Gini proxy at every candidate, the first strict maximum
//      in (visit order, position); random splitter: the class counts at or below its threshold;
//   4. the node's samples partitioned by the best split (stable, team-parallel), the children's impurities and the
//      impurity improvement from their class counts.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

#include "npsum.cuh"

namespace b200aa {
namespace forest {

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsub;

constexpr uint32_t kRandRMax = 2147483647u;                 // RAND_R_MAX (utils/_random.pxd)
constexpr float kFeatureThreshold = 1e-7f;                  // FEATURE_THRESHOLD (tree/_partitioner.pxd), float32
constexpr double kEpsilon = 10 * DBL_EPSILON;               // EPSILON = 10 * np.finfo('double').eps (tree/_criterion.pyx)
constexpr int kMaxClasses = 32;                             // class counts per thread in shared memory
constexpr int kMaxFeats = 512;                              // per-feature state in shared memory
constexpr int kThreads = 128;                               // one CTA per tree
constexpr int32_t kTreeLeaf = -1, kTreeUndefined = -2;      // _TREE_LEAF, _TREE_UNDEFINED

enum Kind { kBest = 0, kRandom = 1 };                      // RandomForestClassifier's splitter / ExtraTreesClassifier's

// our_rand_r, rand_int, rand_uniform (utils/_random.pxd, tree/_utils.pyx)
__host__ __device__ inline uint32_t our_rand_r(uint32_t &s)
{
    if (s == 0) s = 1;
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s % (kRandRMax + 1u);
}
__host__ __device__ inline int64_t rand_int(int64_t lo, int64_t hi, uint32_t &s) { return lo + int64_t(our_rand_r(s)) % (hi - lo); }
__host__ __device__ inline double rand_uniform(double lo, double hi, uint32_t &s)
{
    return dadd(ddiv(dmul(dsub(hi, lo), double(our_rand_r(s))), double(kRandRMax)), lo);
}

__host__ __device__ inline float fadd(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// a feature is constant in a node when max <= min + FEATURE_THRESHOLD, in float32
__host__ __device__ inline bool is_constant(float mn, float mx) { return mx <= fadd(mn, kFeatureThreshold); }
// next_p skips position p of the sorted values while v[p] <= v[p - 1] + FEATURE_THRESHOLD
__host__ __device__ inline bool is_candidate(float prev, float cur) { return !(cur <= fadd(prev, kFeatureThreshold)); }
// the best splitter's threshold: feature_values[p_prev] / 2.0 + feature_values[p] / 2.0
__host__ __device__ inline double mid_threshold(float a, float b) { return dadd(ddiv(double(a), 2.0), ddiv(double(b), 2.0)); }

// Gini of a class-count vector (Gini.node_impurity / children_impurity): 0.0 + (1.0 - sq / (w * w)), sq summed in class
// order; the division by n_outputs = 1 is exact
__host__ __device__ inline double gini(const int64_t *cnt, int C, double w)
{
    double sq = 0.0;
    for (int c = 0; c < C; ++c) sq = dadd(sq, dmul(double(cnt[c]), double(cnt[c])));
    return dadd(0.0, dsub(1.0, ddiv(sq, dmul(w, w))));
}
// the same for the right side of a split: counts total - left
__host__ __device__ inline double gini_rest(const int64_t *total, const int64_t *left, int C, double w)
{
    double sq = 0.0;
    for (int c = 0; c < C; ++c) {
        const double r = double(total[c] - left[c]);
        sq = dadd(sq, dmul(r, r));
    }
    return dadd(0.0, dsub(1.0, ddiv(sq, dmul(w, w))));
}
// Criterion.proxy_impurity_improvement: - w_right * impurity_right - w_left * impurity_left
__host__ __device__ inline double proxy(double wl, double gl, double wr, double gr) { return dsub(dmul(-wr, gr), dmul(wl, gl)); }
// Criterion.impurity_improvement
__host__ __device__ inline double improvement(double w_total, double wn, double imp, double wl, double gl, double wr, double gr)
{
    return dmul(ddiv(wn, w_total), dsub(dsub(imp, dmul(ddiv(wr, wn), gr)), dmul(ddiv(wl, wn), gl)));
}

// float32 bits ordered as the values (-0 before +0, which compare equal and may come in either order)
__host__ __device__ inline uint32_t order_bits(float x)
{
    uint32_t u;
    memcpy(&u, &x, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ inline float from_order_bits(uint32_t o)
{
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    float x;
    memcpy(&x, &u, 4);
    return x;
}

__host__ __device__ inline int64_t pow2_at_least(int64_t n)
{
    int64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}

// max_features="sqrt": max(1, int(np.sqrt(n_features)))
inline int sqrt_features(int F)
{
    int m = int(std::sqrt(double(F)));
    return m < 1 ? 1 : m;
}

// One node of a trained tree as Tree.__getstate__ has it (48 bytes; include/b200aa.h b200aa_forest_node)
struct NodeOut {
    int32_t left, right, feature, n_samples;
    double threshold, impurity, weighted;
    int32_t missing_left, pad;
};
static_assert(sizeof(NodeOut) == 48, "48-byte nodes");

struct StackRec {
    int32_t start, end, depth, parent, is_left, n_const;
    double impurity;
};

// Everything one tree reads and writes.  Global: X, y, w (shared by every tree; w = NULL gives every sample weight 1),
// samples / tmp [n], keys [pow2_at_least(n)], stack [n + 1], nodes [2 n - 1], values [(2 n - 1) C].  Team-shared (shared
// memory on the device): features / constf / drawn [F], mn / mx [F], thr [F], cnt [team size * C], red_proxy / red_pos
// [team size] and st.
struct Shared {
    int64_t node_count, best_nleft, n_drawn, n_const_out, max_depth;
    double best_proxy, best_thr, imp, wn, w_total;
    int32_t best_f, best_k, best_missing_left;
    uint32_t rng;
    int64_t total[kMaxClasses], left[kMaxClasses];
    int32_t stack_top;
};

struct Tree {
    const float *X;
    const int32_t *y, *w;
    int64_t n;
    int F, C, max_features, kind;
    int32_t *samples, *tmp;
    uint64_t *keys;
    StackRec *stack;
    NodeOut *nodes;
    double *values;
    // team-shared
    int32_t *features, *constf, *drawn;
    float *mn, *mx;
    double *thr;
    int64_t *cnt;              // [team size][C]
    double *red_proxy;         // [team size]
    int64_t *red_pos;          // [team size]
    Shared *st;
};

struct Team {
    int tid, n;
    __host__ __device__ void sync() const
    {
#ifdef __CUDA_ARCH__
        __syncthreads();
#endif
    }
};

// Thread 0: the Fisher-Yates draw loop of node_split_best / node_split_random.  Writes the drawn non-constant features in
// visit order to drawn[] (and, for the random splitter, each one's threshold to thr[]), keeps features / constf as
// scikit-learn's splitter keeps them across nodes, and returns the node's n_total_constants.
__host__ __device__ inline int64_t draw_features(int32_t *features, int32_t *constf, int F, int max_features, int kind,
                                                 int64_t n_known, const float *mn, const float *mx, uint32_t &rng,
                                                 int32_t *drawn, double *thr, int64_t &n_drawn)
{
    int64_t f_i = F, n_found = 0, n_drawn_c = 0, n_total = n_known, n_visited = 0;
    n_drawn = 0;
    while (f_i > n_total && (n_visited < max_features || n_visited <= n_found + n_drawn_c)) {
        ++n_visited;
        int64_t f_j = rand_int(n_drawn_c, f_i - n_found, rng);
        if (f_j < n_known) {
            const int32_t t = features[n_drawn_c];
            features[n_drawn_c] = features[f_j];
            features[f_j] = t;
            ++n_drawn_c;
            continue;
        }
        f_j += n_found;
        const int32_t cur = features[f_j];
        if (is_constant(mn[cur], mx[cur])) {
            features[f_j] = features[n_total];
            features[n_total] = cur;
            ++n_found;
            ++n_total;
            continue;
        }
        --f_i;
        features[f_j] = features[f_i];
        features[f_i] = cur;
        drawn[n_drawn] = cur;
        if (kind == kRandom) {
            double t = rand_uniform(double(mn[cur]), double(mx[cur]), rng);
            if (t == double(mx[cur])) t = double(mn[cur]);
            thr[n_drawn] = t;
        }
        ++n_drawn;
    }
    for (int64_t i = 0; i < n_known; ++i) features[i] = constf[i];
    for (int64_t i = 0; i < n_found; ++i) constf[n_known + i] = features[n_known + i];
    return n_total;
}

// class counts of samples[lo, hi) into the team's per-thread rows, then summed per class into out (exact integers)
__host__ __device__ inline void class_counts(const Tree &T, const Team &tm, int64_t lo, int64_t hi, const float *xf_or_null,
                                             int f, double threshold, int64_t *out, int64_t *n_out)
{
    int64_t *mine = T.cnt + int64_t(tm.tid) * T.C;
    for (int c = 0; c < T.C; ++c) mine[c] = 0;
    int64_t k = 0;
    for (int64_t p = lo + tm.tid; p < hi; p += tm.n) {
        const int32_t s = T.samples[p];
        if (xf_or_null && !(double(xf_or_null[int64_t(s) * T.F + f]) <= threshold)) continue;
        mine[T.y[s]] += T.w ? T.w[s] : 1;
        ++k;
    }
    T.red_pos[tm.tid] = k;
    tm.sync();
    if (tm.tid == 0) {
        int64_t kk = 0;
        for (int t = 0; t < tm.n; ++t) kk += T.red_pos[t];
        *n_out = kk;
    }
    for (int c = tm.tid; c < T.C; c += tm.n) {
        int64_t a = 0;
        for (int t = 0; t < tm.n; ++t) a += T.cnt[int64_t(t) * T.C + c];
        out[c] = a;
    }
    tm.sync();
}

// sum of a class-count vector as the criterion's weighted_n (exact)
__host__ __device__ inline double weight_of(const int64_t *cnt, int C)
{
    int64_t a = 0;
    for (int c = 0; c < C; ++c) a += cnt[c];
    return double(a);
}

// Best splitter, one feature f over samples[lo, hi): sort, then every candidate's proxy; the first strict maximum of this
// feature goes to st->best_* when it beats the best so far.
__host__ __device__ inline void eval_best(const Tree &T, const Team &tm, int64_t lo, int64_t hi, int f, int k)
{
    Shared &S = *T.st;
    const int64_t m = hi - lo, m2 = pow2_at_least(m);
    for (int64_t i = tm.tid; i < m2; i += tm.n) {
        if (i < m) {
            const int32_t s = T.samples[lo + i];
            T.keys[i] = (uint64_t(order_bits(T.X[int64_t(s) * T.F + f])) << 32) | uint32_t(s);
        } else {
            T.keys[i] = ~uint64_t(0);
        }
    }
    tm.sync();
    for (int64_t kk = 2; kk <= m2; kk <<= 1) {
        for (int64_t j = kk >> 1; j > 0; j >>= 1) {
            for (int64_t i = tm.tid; i < m2; i += tm.n) {
                const int64_t l = i ^ j;
                if (l > i) {
                    const uint64_t a = T.keys[i], b = T.keys[l];
                    if ((a > b) == ((i & kk) == 0)) {
                        T.keys[i] = b;
                        T.keys[l] = a;
                    }
                }
            }
            tm.sync();
        }
    }
    // chunk of positions per thread, the class counts of every earlier chunk as its start
    const int64_t chunk = (m + tm.n - 1) / tm.n, q0 = tm.tid * chunk, q1 = q0 + chunk < m ? q0 + chunk : m;
    int64_t *mine = T.cnt + int64_t(tm.tid) * T.C;
    for (int c = 0; c < T.C; ++c) mine[c] = 0;
    for (int64_t q = q0; q < q1; ++q) {
        const int32_t s = int32_t(uint32_t(T.keys[q]));
        mine[T.y[s]] += T.w ? T.w[s] : 1;
    }
    tm.sync();
    int64_t run[kMaxClasses];
    for (int c = 0; c < T.C; ++c) {
        int64_t a = 0;
        for (int t = 0; t < tm.tid; ++t) a += T.cnt[int64_t(t) * T.C + c];
        run[c] = a;
    }
    const double wn = S.wn;
    double bp = -INFINITY;
    int64_t bq = -1;
    for (int64_t q = q0; q < q1; ++q) {
        if (q >= 1 && is_candidate(from_order_bits(uint32_t(T.keys[q - 1] >> 32)), from_order_bits(uint32_t(T.keys[q] >> 32)))) {
            const double wl = weight_of(run, T.C), wr = dsub(wn, wl);
            const double pr = proxy(wl, gini(run, T.C, wl), wr, gini_rest(S.total, run, T.C, wr));
            if (pr > bp) {
                bp = pr;
                bq = q;
            }
        }
        const int32_t s = int32_t(uint32_t(T.keys[q]));
        run[T.y[s]] += T.w ? T.w[s] : 1;
    }
    T.red_proxy[tm.tid] = bp;
    T.red_pos[tm.tid] = bq;
    tm.sync();
    if (tm.tid == 0) {
        double fp = -INFINITY;
        int64_t fq = -1;
        for (int t = 0; t < tm.n; ++t)
            if (T.red_pos[t] >= 0 && T.red_proxy[t] > fp) {
                fp = T.red_proxy[t];
                fq = T.red_pos[t];
            }
        if (fq >= 0 && fp > S.best_proxy) {
            S.best_proxy = fp;
            S.best_f = f;
            S.best_k = k;
            S.best_nleft = fq;
            S.best_thr = mid_threshold(from_order_bits(uint32_t(T.keys[fq - 1] >> 32)), from_order_bits(uint32_t(T.keys[fq] >> 32)));
            S.best_missing_left = fq > m - fq;
        }
    }
    tm.sync();
}

// Random splitter, one drawn feature f with its threshold: the counts at or below it and the proxy
__host__ __device__ inline void eval_random(const Tree &T, const Team &tm, int64_t lo, int64_t hi, int f, int k, double t)
{
    Shared &S = *T.st;
    int64_t n_left = 0;
    class_counts(T, tm, lo, hi, T.X, f, t, S.left, &n_left);
    if (tm.tid == 0) {
        const int64_t n_right = (hi - lo) - n_left;
        if (n_left >= 1 && n_right >= 1) {
            const double wl = weight_of(S.left, T.C), wr = dsub(S.wn, wl);
            const double pr = proxy(wl, gini(S.left, T.C, wl), wr, gini_rest(S.total, S.left, T.C, wr));
            if (pr > S.best_proxy) {
                S.best_proxy = pr;
                S.best_f = f;
                S.best_k = k;
                S.best_nleft = n_left;
                S.best_thr = t;
                S.best_missing_left = n_left > n_right;
            }
        }
    }
    tm.sync();
}

// Stable partition of samples[lo, hi) by x[f] <= t through tmp: each thread's chunk, its left / right counts placed after
// every earlier chunk's
__host__ __device__ inline void partition(const Tree &T, const Team &tm, int64_t lo, int64_t hi, int f, double t, int64_t n_left)
{
    const int64_t m = hi - lo, chunk = (m + tm.n - 1) / tm.n, q0 = lo + tm.tid * chunk;
    const int64_t q1 = q0 + chunk < hi ? q0 + chunk : hi;
    int64_t l = 0;
    for (int64_t q = q0; q < q1; ++q) l += double(T.X[int64_t(T.samples[q]) * T.F + f]) <= t;
    T.red_pos[tm.tid] = l;
    tm.sync();
    int64_t lb = 0, rb = 0;
    for (int t2 = 0; t2 < tm.tid; ++t2) {
        const int64_t a0 = lo + t2 * chunk, a1 = a0 + chunk < hi ? a0 + chunk : hi;
        const int64_t len = a1 > a0 ? a1 - a0 : 0;
        lb += T.red_pos[t2];
        rb += len - T.red_pos[t2];
    }
    int64_t li = lo + lb, ri = lo + n_left + rb;
    for (int64_t q = q0; q < q1; ++q) {
        const int32_t s = T.samples[q];
        if (double(T.X[int64_t(s) * T.F + f]) <= t) T.tmp[li++] = s;
        else T.tmp[ri++] = s;
    }
    tm.sync();
    for (int64_t q = lo + tm.tid; q < hi; q += tm.n) T.samples[q] = T.tmp[q];
    tm.sync();
}

// The whole tree: DepthFirstTreeBuilder.build with the library's parameters.  rand_r_seed: the splitter's rand_r_state
// (RandomState(tree seed).randint(0, RAND_R_MAX)).  Writes nodes / values and st->node_count, st->max_depth.
__host__ __device__ inline void build_tree(const Tree &T, const Team &tm, uint32_t rand_r_seed)
{
    Shared &S = *T.st;
    // Splitter.init: the positively weighted samples in index order, weighted_n_samples over every sample
    if (tm.tid == 0) {
        int64_t j = 0, wt = 0;
        for (int64_t i = 0; i < T.n; ++i) {
            const int32_t wi = T.w ? T.w[i] : 1;
            if (wi != 0) T.samples[j++] = int32_t(i);
            wt += wi;
        }
        S.w_total = double(wt);
        S.rng = rand_r_seed;
        S.node_count = 0;
        S.max_depth = -1;
        S.stack_top = 1;
        T.stack[0] = StackRec{0, int32_t(j), 0, kTreeUndefined, 0, 0, INFINITY};
    }
    for (int f = tm.tid; f < T.F; f += tm.n) T.features[f] = f;
    tm.sync();
    bool first = true;
    while (S.stack_top > 0) {
        const StackRec rec = T.stack[S.stack_top - 1];
        tm.sync();
        const int64_t lo = rec.start, hi = rec.end, m = hi - lo;
        int64_t nn = 0;
        class_counts(T, tm, lo, hi, nullptr, 0, 0.0, S.total, &nn);
        if (tm.tid == 0) {
            S.stack_top -= 1;
            S.wn = weight_of(S.total, T.C);
            S.imp = first ? gini(S.total, T.C, S.wn) : rec.impurity;
            S.best_proxy = -INFINITY;
            S.best_k = -1;
            S.n_drawn = 0;
        }
        first = false;
        tm.sync();
        bool leaf = m < 2 || S.imp <= kEpsilon;
        if (!leaf) {
            for (int f = tm.tid; f < T.F; f += tm.n) {
                float a = T.X[int64_t(T.samples[lo]) * T.F + f], b = a;
                for (int64_t p = lo + 1; p < hi; ++p) {
                    const float v = T.X[int64_t(T.samples[p]) * T.F + f];
                    if (v < a) a = v;
                    else if (v > b) b = v;
                }
                T.mn[f] = a;
                T.mx[f] = b;
            }
            tm.sync();
            if (tm.tid == 0) {
                int64_t nd = 0;
                S.n_const_out = draw_features(T.features, T.constf, T.F, T.max_features, T.kind, rec.n_const, T.mn, T.mx, S.rng,
                                              T.drawn, T.thr, nd);
                S.n_drawn = nd;
            }
            tm.sync();
            const int64_t nd = S.n_drawn;
            for (int64_t k = 0; k < nd; ++k) {
                if (T.kind == kBest) eval_best(T, tm, lo, hi, T.drawn[k], int(k));
                else eval_random(T, tm, lo, hi, T.drawn[k], int(k), T.thr[k]);
            }
            double gl = 0.0, gr = 0.0;
            if (S.best_k >= 0) {
                partition(T, tm, lo, hi, S.best_f, S.best_thr, S.best_nleft);
                int64_t nl = 0;
                class_counts(T, tm, lo, lo + S.best_nleft, nullptr, 0, 0.0, S.left, &nl);
                const double wl = weight_of(S.left, T.C), wr = dsub(S.wn, wl);
                gl = gini(S.left, T.C, wl);
                gr = gini_rest(S.total, S.left, T.C, wr);
                const double impr = improvement(S.w_total, S.wn, S.imp, wl, gl, wr, gr);
                leaf = impr + kEpsilon < 0.0;
            } else {
                leaf = true;
            }
            if (tm.tid == 0 && !leaf) {
                const int32_t pos = int32_t(lo + S.best_nleft), d = rec.depth + 1, id = int32_t(S.node_count);
                const int32_t nc = int32_t(S.n_const_out);
                T.stack[S.stack_top++] = StackRec{pos, int32_t(hi), d, id, 0, nc, gr};
                T.stack[S.stack_top++] = StackRec{int32_t(lo), pos, d, id, 1, nc, gl};
            }
        }
        if (tm.tid == 0) {
            const int64_t id = S.node_count++;
            NodeOut &o = T.nodes[id];
            o.n_samples = int32_t(m);
            o.impurity = S.imp;
            o.weighted = S.wn;
            o.pad = 0;
            if (leaf) {
                o.left = o.right = kTreeLeaf;
                o.feature = kTreeUndefined;
                o.threshold = double(kTreeUndefined);
                o.missing_left = 0;
            } else {
                o.left = o.right = 0;           // set when the children are added
                o.feature = S.best_f;
                o.threshold = S.best_thr;
                o.missing_left = S.best_missing_left;
            }
            if (rec.parent != kTreeUndefined) {
                if (rec.is_left) T.nodes[rec.parent].left = int32_t(id);
                else T.nodes[rec.parent].right = int32_t(id);
            }
            for (int c = 0; c < T.C; ++c) T.values[id * T.C + c] = ddiv(double(S.total[c]), S.wn);
            if (rec.depth > S.max_depth) S.max_depth = rec.depth;
        }
        tm.sync();
    }
}

}  // namespace forest
}  // namespace b200aa
