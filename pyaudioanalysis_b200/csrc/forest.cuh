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
// CTA (Team = the block, sync = __syncthreads), in tests/forest_host.cu a team of std::threads on the CPU.  Per node:
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

#include "front.cuh"
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

// Dynamic shared memory of forest_build_kernel (csrc/forest.cu): st, thr [F], cnt [kThreads C], red_proxy / red_pos
// [kThreads], mn / mx / features / constf / drawn [F].  Every launcher sets the kernel's attribute to kSmemCap, the size at
// the largest shape it accepts, never to its own call's size: a thread setting a smaller size between another thread's
// set and launch would make that launch fail.
constexpr size_t smem_bytes(int F, int C)
{
    return sizeof(Shared) + size_t(F) * (3 * 4 + 2 * 4 + 8) + size_t(kThreads) * (size_t(C) * 8 + 16) + 64;
}
constexpr size_t kSmemCap = smem_bytes(kMaxFeats, kMaxClasses);

// forest_build_kernel's dynamic shared memory at s (16-aligned) carved into T's team-shared arrays for a team of `team`
// threads, in the order smem_bytes counts them (T.F and T.C set).  Returns the end of the carve.
__host__ __device__ inline unsigned char *carve_smem(unsigned char *s, size_t team, Tree &T)
{
    T.st = reinterpret_cast<Shared *>(s);
    s += (sizeof(Shared) + 15) & ~size_t(15);
    T.thr = reinterpret_cast<double *>(s);
    s += size_t(T.F) * 8;
    T.cnt = reinterpret_cast<int64_t *>(s);
    s += team * T.C * 8;
    T.red_proxy = reinterpret_cast<double *>(s);
    s += team * 8;
    T.red_pos = reinterpret_cast<int64_t *>(s);
    s += team * 8;
    T.mn = reinterpret_cast<float *>(s);
    T.mx = T.mn + T.F;
    T.features = reinterpret_cast<int32_t *>(T.mx + T.F);
    T.constf = T.features + T.F;
    T.drawn = T.constf + T.F;
    return reinterpret_cast<unsigned char *>(T.drawn + T.F);
}

// The team building one tree: on the device the CTA (sync = __syncthreads); on the host, tid / n of threads that meet at
// wait(wait_ctx), a barrier (tests/ run the builders on std::threads), or a team of one with no wait.
struct Team {
    int tid, n;
    void (*wait)(void *) = nullptr;
    void *wait_ctx = nullptr;
    __host__ __device__ void sync() const
    {
#ifdef __CUDA_ARCH__
        __syncthreads();
#else
        if (wait) wait(wait_ctx);
#endif
    }
};

// Thread 0: the Fisher-Yates draw loop of node_split_best / node_split_random.  Writes the drawn non-constant features in
// visit order to drawn[] (and, for the random splitter, each one's threshold to thr[]), keeps features / constf as
// scikit-learn's splitter keeps them across nodes, and returns the node's n_total_constants.  With `visited`, it also
// writes every feature the best splitter sorts, in visit order: the drawn non-constant ones and the ones found constant
// (not those drawn from the known-constant range), and their number to n_visited_out (the regressor needs the sort order
// each of them leaves).
__host__ __device__ inline int64_t draw_features(int32_t *features, int32_t *constf, int F, int max_features, int kind,
                                                 int64_t n_known, const float *mn, const float *mx, uint32_t &rng,
                                                 int32_t *drawn, double *thr, int64_t &n_drawn,
                                                 int32_t *visited = nullptr, int64_t *n_visited_out = nullptr)
{
    int64_t f_i = F, n_found = 0, n_drawn_c = 0, n_total = n_known, n_visited = 0, n_sorted = 0;
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
        if (visited) visited[n_sorted++] = cur;
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
    if (n_visited_out) *n_visited_out = n_sorted;
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

// ------------------------------------------------------------------------------------------------
// Regression: RandomForestRegressor(n_estimators=T).fit with the library's arguments (criterion="squared_error",
// max_features=1.0, bootstrap, min_samples_split=2, min_samples_leaf=1, no depth limit), node for node, bit for bit.
//
// A regressor's node sums are float64 sums of w * y, so they depend on the order of samples[start:end] at every step,
// and that order is the one scikit-learn's splitter leaves:
//   - node_split_best sorts every visited feature's values in place together with samples[start:end] by introsort_3way
//     (utils/_sorting.pyx simultaneous_sort, use_three_way_partition=True), each sort starting from the order the
//     previous one left ("visited" includes a feature then found constant, not one drawn from the known-constant range);
//   - partition_samples_final, a swap partition, starts from the order the last visited feature left.
// Where a feature's values in the node are pairwise different (-0 == +0 counts as equal), the sorted order is unique and
// any sort gives it; otherwise introsort_3way is replayed from the order it starts from.
//
// The criterion (tree/_criterion.pyx RegressionCriterion / MSE), every sum sequential in the samples' order:
//   init:    sum_total += w*y, sq_sum_total += (w*y)*y, weighted_n += w over samples[start:end]
//   update(new_pos), called only at candidate positions: forward (sum_left += w*y from pos) when new_pos - pos <=
//            end - new_pos, else reverse_reset (sum_left = sum_total) and sum_left -= w*y from end - 1 down to new_pos
//   proxy:   sl*sl / wl + sr*sr / wr, sr = sum_total - sl
//   after the best split: the partition, reset, update(best.pos) over the partitioned order, children_impurity
//            (sq_sum_left += (w*y)*y over samples[start:pos]) and impurity_improvement.
// Node values are sum_total / weighted_n.  The leaf tests use tree/_tree.pyx's EPSILON = np.finfo('double').eps.
//
// build_regression_tree() runs it for a team of threads.  Per node: the node's sums (thread 0, in order); every feature's
// min / max; the Fisher-Yates draw (draw_features, recording the visits); every visit's (value, sample) keys sorted at
// once by one batched bitonic sort (team-parallel); ties detected (team-parallel); thread 0 replays introsort_3way, in
// visit order, for the visits with ties only; one candidate chain per visit, each on its own thread; thread 0 takes the
// first strict maximum in (visit order, position), partitions, and computes the children's impurities.
constexpr double kLeafEpsilon = DBL_EPSILON;                // EPSILON of tree/_tree.pyx

// ---- introsort_3way (utils/_sorting.pyx), on float32 values with int32 sample indices ----
__host__ __device__ inline void sort_swap(float *v, int32_t *ix, int64_t i, int64_t j)
{
    const float tv = v[i];
    v[i] = v[j];
    v[j] = tv;
    const int32_t ti = ix[i];
    ix[i] = ix[j];
    ix[j] = ti;
}
__host__ __device__ inline float median3(const float *v, int64_t n)
{
    const float a = v[0], b = v[n / 2], c = v[n - 1];
    if (a < b) {
        if (b < c) return b;
        if (a < c) return c;
        return a;
    }
    if (b < c) {
        if (a < c) return a;
        return c;
    }
    return b;
}
__host__ __device__ inline void insertion_sort(float *v, int32_t *ix, int64_t n)
{
    for (int64_t i = 1; i < n; ++i) {
        const float tv = v[i];
        const int32_t ti = ix[i];
        int64_t j = i;
        while (j > 0 && v[j - 1] > tv) {
            v[j] = v[j - 1];
            ix[j] = ix[j - 1];
            --j;
        }
        v[j] = tv;
        ix[j] = ti;
    }
}
__host__ __device__ inline void sift_down(float *v, int32_t *ix, int64_t start, int64_t end)
{
    int64_t root = start;
    while (true) {
        const int64_t child = root * 2 + 1;
        int64_t maxind = root;
        if (child < end && v[maxind] < v[child]) maxind = child;
        if (child + 1 < end && v[maxind] < v[child + 1]) maxind = child + 1;
        if (maxind == root) break;
        sort_swap(v, ix, root, maxind);
        root = maxind;
    }
}
__host__ __device__ inline void heapsort(float *v, int32_t *ix, int64_t n)
{
    int64_t start = (n - 2) / 2, end = n;        // n > 15 here: C's and Python's integer division agree
    while (true) {
        sift_down(v, ix, start, end);
        if (start == 0) break;
        --start;
    }
    end = n - 1;
    while (end > 0) {
        sort_swap(v, ix, 0, end);
        sift_down(v, ix, 0, end);
        --end;
    }
}
// floor(log2(n)) for n >= 1.  simultaneous_sort takes maxd = 2 * (intp)log2(n) with libm's log2; for n < 2^29 they agree:
// log2(n) is exact at a power of two, and otherwise lies in (k, k + 1) at least log2(2^(k+1)) - log2(2^(k+1) - 1) >
// 2^-(k+1) / ln 2 >= 2^-29 / ln 2 ~ 2.7e-9 below k + 1, a gap a million times an ulp of a number below 32 (3.6e-15), so
// a log2 correct to within an ulp cannot reach k + 1 and truncates to k.
__host__ __device__ inline int64_t floor_log2(int64_t n)
{
    int64_t k = 0;
    while ((n >> (k + 1)) != 0) ++k;
    return k;
}
// simultaneous_sort(values, indices, n, use_three_way_partition=True).  introsort_3way recurses on the left part and
// loops on the right one; the parts are disjoint and each one's sort depends only on its own contents and depth budget,
// so an explicit stack of pending (offset, length, maxd) parts gives the same result.  Pending parts <= the initial maxd.
__host__ __device__ inline void introsort_3way(float *v, int32_t *ix, int64_t n)
{
    if (n == 0) return;
    struct Part {
        int64_t off, n, maxd;
    };
    Part stack[64];
    int top = 0;
    stack[top++] = Part{0, n, 2 * floor_log2(n)};
    while (top > 0) {
        Part p = stack[--top];
        float *pv = v + p.off;
        int32_t *pi = ix + p.off;
        bool done = false;
        while (p.n > 15) {
            if (p.maxd <= 0) {
                heapsort(pv, pi, p.n);
                done = true;
                break;
            }
            --p.maxd;
            const float pivot = median3(pv, p.n);
            int64_t i = 0, l = 0, r = p.n;
            while (i < r) {
                if (pv[i] < pivot) {
                    sort_swap(pv, pi, i, l);
                    ++i;
                    ++l;
                } else if (pv[i] > pivot) {
                    --r;
                    sort_swap(pv, pi, i, r);
                } else {
                    ++i;
                }
            }
            stack[top++] = Part{p.off, l, p.maxd};
            p.off += r;
            pv += r;
            pi += r;
            p.n -= r;
        }
        if (!done) insertion_sort(pv, pi, p.n);
    }
}

// partition_samples_final (tree/_partitioner.pyx): the swap partition of samples[0, m) by x <= threshold
template <class Xf>
__host__ __device__ inline void swap_partition(int32_t *samples, int64_t m, const Xf &x, double threshold)
{
    int64_t ps = 0, pe = m;
    while (ps < pe) {
        if (double(x(samples[ps])) <= threshold) {
            ++ps;
        } else {
            --pe;
            const int32_t t = samples[ps];
            samples[ps] = samples[pe];
            samples[pe] = t;
        }
    }
}

struct RegShared {
    int64_t node_count, max_depth, n_vis, n_drawn, n_const_out, best_pos;
    double best_proxy, best_thr, imp, wn, w_total, sum_total, sq_total, imp_left, imp_right;
    int32_t best_v, best_f, best_missing_left, leaf, stack_top;
    uint32_t rng;
};

// Everything one regression tree reads and writes.  Global: X [rows, F] and y [rows] (shared by every tree; rows[s] is
// local sample s's row, or s when rows is NULL), w [n] (bootstrap counts), samples / idx [n] and fv [n] (the replay's
// indices and values), keys [F * pow2_at_least(n)], stack [n + 1], nodes [2 n - 1], values [2 n - 1].  Team-shared:
// features / constf / drawn / vis / tied [F], mn / mx [F], vproxy / vpos [F] and st.
struct RegTree {
    const float *X;
    const double *y;
    const int32_t *rows, *w;
    int64_t n;
    int F;
    int32_t *samples, *idx;
    float *fv;
    uint64_t *keys;
    StackRec *stack;
    NodeOut *nodes;
    double *values;
    int32_t *features, *constf, *drawn, *vis, *tied;
    float *mn, *mx;
    double *vproxy;
    int64_t *vpos;
    RegShared *st;
    // y_stride 0: the target of local sample s is y[row(s)] (the forest's targets of every row); else y[s * y_stride]
    // (gradient boosting: column k of the problem's [n, K] negative gradients)
    int32_t y_stride = 0;
    // DepthFirstTreeBuilder's max_depth: the forest has none (np.iinfo(np.int32).max), gradient boosting 3
    int32_t max_depth = INT32_MAX;
    __host__ __device__ int64_t row(int32_t s) const { return rows ? int64_t(rows[s]) : int64_t(s); }
    __host__ __device__ float x(int32_t s, int f) const { return X[row(s) * F + f]; }
    __host__ __device__ double yv(int32_t s) const { return y_stride ? y[int64_t(s) * y_stride] : y[row(s)]; }
    __host__ __device__ double wv(int32_t s) const { return double(w[s]); }
};

// Dynamic shared memory of forest_reg_build_kernel: st, vproxy / vpos [F], mn / mx / features / constf / drawn / vis /
// tied [F]; the attribute is set to kRegSmemCap (as kSmemCap)
constexpr size_t reg_smem_bytes(int F) { return sizeof(RegShared) + size_t(F) * (5 * 4 + 2 * 4 + 16) + 64; }
constexpr size_t kRegSmemCap = reg_smem_bytes(kMaxFeats);

// forest_reg_build_kernel's dynamic shared memory at s (16-aligned) carved into T's team-shared arrays, in the order
// reg_smem_bytes counts them (T.F set).  Returns the end of the carve.  boost_build_kernel carves the same with part
// [kThreads] after vpos (boost_smem_bytes).
__host__ __device__ inline unsigned char *carve_reg_smem(unsigned char *s, RegTree &T)
{
    T.st = reinterpret_cast<RegShared *>(s);
    s += (sizeof(RegShared) + 15) & ~size_t(15);
    T.vproxy = reinterpret_cast<double *>(s);
    s += size_t(T.F) * 8;
    T.vpos = reinterpret_cast<int64_t *>(s);
    s += size_t(T.F) * 8;
    T.mn = reinterpret_cast<float *>(s);
    T.mx = T.mn + T.F;
    T.features = reinterpret_cast<int32_t *>(T.mx + T.F);
    T.constf = T.features + T.F;
    T.drawn = T.constf + T.F;
    T.vis = T.drawn + T.F;
    T.tied = T.vis + T.F;
    return reinterpret_cast<unsigned char *>(T.tied + T.F);
}

// Sets a flag that several of the team's threads may set between two syncs: a plain store on the device, a relaxed
// atomic one on the host, where concurrent plain stores (even of one value) are a data race to C++ and ThreadSanitizer.
__host__ __device__ inline void set_flag(int32_t &f)
{
#ifdef __CUDA_ARCH__
    f = 1;
#else
    __atomic_store_n(&f, 1, __ATOMIC_RELAXED);
#endif
}

__host__ __device__ inline uint64_t reg_key(float v, int32_t s) { return (uint64_t(order_bits(v)) << 32) | uint32_t(s); }
__host__ __device__ inline float key_value(uint64_t k) { return from_order_bits(uint32_t(k >> 32)); }
__host__ __device__ inline int32_t key_sample(uint64_t k) { return int32_t(uint32_t(k)); }

// The regressor's criterion at a split position of one sample order: sum_left and weighted_n_left after reset and
// update(pos) from the current (pos0, sl, wl), forward or from the end as RegressionCriterion.update chooses.
template <class Sample>
__host__ __device__ inline void reg_update(const RegTree &T, const Sample &sample, int64_t m, double sum_total, double wn,
                                           int64_t &pos, double &sl, double &wl, int64_t new_pos)
{
    if (new_pos - pos <= m - new_pos) {
        for (int64_t p = pos; p < new_pos; ++p) {
            const int32_t s = sample(p);
            const double w = T.wv(s);
            sl = dadd(sl, dmul(w, T.yv(s)));
            wl = dadd(wl, w);
        }
    } else {
        sl = sum_total;                 // reverse_reset
        wl = wn;
        for (int64_t p = m - 1; p >= new_pos; --p) {
            const int32_t s = sample(p);
            const double w = T.wv(s);
            sl = dsub(sl, dmul(w, T.yv(s)));
            wl = dsub(wl, w);
        }
    }
    pos = new_pos;
}
// MSE.proxy_impurity_improvement
__host__ __device__ inline double reg_proxy(double sl, double wl, double sr, double wr)
{
    return dadd(ddiv(dadd(0.0, dmul(sl, sl)), wl), ddiv(dadd(0.0, dmul(sr, sr)), wr));
}
__host__ __device__ inline double square(double a) { return dmul(a, a); }     // Cython's a ** 2.0 folds to a * a

// One visit's candidate chain over its sorted keys K[0, m): the first strict maximum of the proxy, or bq = -1 when the
// feature has no candidate.
__host__ __device__ inline void reg_chain(const RegTree &T, const uint64_t *K, int64_t m, double sum_total, double wn,
                                          double &bp, int64_t &bq)
{
    const auto sample = [K](int64_t p) { return key_sample(K[p]); };
    int64_t pos = 0;
    double sl = 0.0, wl = 0.0;                 // reset
    bp = -INFINITY;
    bq = -1;
    float prev = key_value(K[0]);
    for (int64_t q = 1; q < m; ++q) {
        const float cur = key_value(K[q]);
        if (is_candidate(prev, cur)) {
            reg_update(T, sample, m, sum_total, wn, pos, sl, wl, q);
            const double proxy_q = reg_proxy(sl, wl, dsub(sum_total, sl), dsub(wn, wl));
            if (proxy_q > bp) {
                bp = proxy_q;
                bq = q;
            }
        }
        prev = cur;
    }
}

// The whole tree: DepthFirstTreeBuilder.build with the regressor's parameters.  rand_r_seed: the splitter's
// rand_r_state.  Writes nodes / values (one per node) and st->node_count, st->max_depth.
__host__ __device__ inline void build_regression_tree(const RegTree &T, const Team &tm, uint32_t rand_r_seed)
{
    RegShared &S = *T.st;
    if (tm.tid == 0) {
        int64_t j = 0, wt = 0;
        for (int64_t i = 0; i < T.n; ++i) {
            if (T.w[i] != 0) T.samples[j++] = int32_t(i);
            wt += T.w[i];
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
        int32_t *smp = T.samples + lo;
        if (tm.tid == 0) {
            S.stack_top -= 1;
            // node_reset -> criterion.init, in the node's current order
            double st_ = 0.0, sq = 0.0, wn = 0.0;
            for (int64_t p = 0; p < m; ++p) {
                const int32_t s = smp[p];
                const double w = T.wv(s), wy = dmul(w, T.yv(s));
                st_ = dadd(st_, wy);
                sq = dadd(sq, dmul(wy, T.yv(s)));
                wn = dadd(wn, w);
            }
            S.sum_total = st_;
            S.sq_total = sq;
            S.wn = wn;
            S.imp = first ? dsub(ddiv(sq, wn), square(ddiv(st_, wn))) : rec.impurity;
            S.best_proxy = -INFINITY;
            S.best_v = -1;
            S.n_vis = 0;
            S.leaf = rec.depth >= T.max_depth || m < 2 || S.imp <= kLeafEpsilon;
        }
        first = false;
        tm.sync();
        if (!S.leaf) {
            for (int f = tm.tid; f < T.F; f += tm.n) {
                float a = T.x(smp[0], f), b = a;
                for (int64_t p = 1; p < m; ++p) {
                    const float v = T.x(smp[p], f);
                    if (v < a) a = v;
                    else if (v > b) b = v;
                }
                T.mn[f] = a;
                T.mx[f] = b;
            }
            tm.sync();
            if (tm.tid == 0) {
                int64_t nd = 0, nv = 0;
                S.n_const_out = draw_features(T.features, T.constf, T.F, T.F, kBest, rec.n_const, T.mn, T.mx, S.rng, T.drawn,
                                              nullptr, nd, T.vis, &nv);
                S.n_drawn = nd;
                S.n_vis = nv;
            }
            tm.sync();
            const int64_t nv = S.n_vis, m2 = pow2_at_least(m);
            // every visit's keys, sorted at once: segment v is keys[v m2, (v + 1) m2), padded with keys above any value
            for (int64_t i = tm.tid; i < nv * m2; i += tm.n) {
                const int64_t v = i / m2, q = i - v * m2;
                T.keys[i] = q < m ? reg_key(T.x(smp[q], T.vis[v]), smp[q]) : ~uint64_t(0);
            }
            for (int64_t v = tm.tid; v < nv; v += tm.n) T.tied[v] = 0;
            tm.sync();
            for (int64_t kk = 2; kk <= m2; kk <<= 1) {
                for (int64_t j = kk >> 1; j > 0; j >>= 1) {
                    for (int64_t i = tm.tid; i < nv * m2; i += tm.n) {
                        const int64_t q = i & (m2 - 1), l = q ^ j;
                        if (l > q) {
                            uint64_t *seg = T.keys + (i - q);
                            const uint64_t a = seg[q], b = seg[l];
                            if ((a > b) == ((q & kk) == 0)) {
                                seg[q] = b;
                                seg[l] = a;
                            }
                        }
                    }
                    tm.sync();
                }
            }
            for (int64_t i = tm.tid; i < nv * m; i += tm.n) {
                const int64_t v = i / m, q = i - v * m;
                if (q >= 1 && key_value(T.keys[v * m2 + q - 1]) == key_value(T.keys[v * m2 + q])) set_flag(T.tied[v]);
            }
            tm.sync();
            // introsort_3way replayed for the visits with ties, in visit order, each from the order the one before left
            if (tm.tid == 0) {
                for (int64_t v = 0; v < nv; ++v) {
                    if (!T.tied[v]) continue;
                    const int f = T.vis[v];
                    for (int64_t q = 0; q < m; ++q) {
                        const int32_t s = v == 0 ? smp[q] : key_sample(T.keys[(v - 1) * m2 + q]);
                        T.idx[q] = s;
                        T.fv[q] = T.x(s, f);
                    }
                    introsort_3way(T.fv, T.idx, m);
                    for (int64_t q = 0; q < m; ++q) T.keys[v * m2 + q] = reg_key(T.fv[q], T.idx[q]);
                }
            }
            tm.sync();
            // one candidate chain per visit; a visit found constant has no candidate
            for (int64_t v = tm.tid; v < nv; v += tm.n) {
                const int f = T.vis[v];
                double bp = -INFINITY;
                int64_t bq = -1;
                if (!is_constant(T.mn[f], T.mx[f])) reg_chain(T, T.keys + v * m2, m, S.sum_total, S.wn, bp, bq);
                T.vproxy[v] = bp;
                T.vpos[v] = bq;
            }
            tm.sync();
            if (tm.tid == 0) {
                for (int64_t v = 0; v < nv; ++v)
                    if (T.vpos[v] >= 0 && T.vproxy[v] > S.best_proxy) {
                        const uint64_t *K = T.keys + v * m2;
                        const int64_t q = T.vpos[v];
                        S.best_proxy = T.vproxy[v];
                        S.best_v = int32_t(v);
                        S.best_f = T.vis[v];
                        S.best_pos = q;
                        S.best_thr = mid_threshold(key_value(K[q - 1]), key_value(K[q]));
                        S.best_missing_left = q > m - q;
                    }
                if (S.best_v < 0) {
                    S.leaf = 1;
                } else {
                    // partition_samples_final from the order the last visit left, then reset, update(best.pos) and
                    // children_impurity over the partitioned order
                    for (int64_t q = 0; q < m; ++q) smp[q] = key_sample(T.keys[(nv - 1) * m2 + q]);
                    const int bf = S.best_f;
                    swap_partition(smp, m, [&T, bf](int32_t s) { return T.x(s, bf); }, S.best_thr);
                    const int64_t pos = S.best_pos;
                    int64_t p0 = 0;
                    double sl = 0.0, wl = 0.0;
                    reg_update(T, [smp](int64_t p) { return smp[p]; }, m, S.sum_total, S.wn, p0, sl, wl, pos);
                    double sq_left = 0.0;
                    for (int64_t p = 0; p < pos; ++p) {
                        const int32_t s = smp[p];
                        sq_left = dadd(sq_left, dmul(dmul(T.wv(s), T.yv(s)), T.yv(s)));
                    }
                    const double wr = dsub(S.wn, wl), sr = dsub(S.sum_total, sl);
                    const double gl = dsub(ddiv(sq_left, wl), square(ddiv(sl, wl)));
                    const double gr = dsub(ddiv(dsub(S.sq_total, sq_left), wr), square(ddiv(sr, wr)));
                    const double impr = improvement(S.w_total, S.wn, S.imp, wl, gl, wr, gr);
                    S.leaf = dadd(impr, kLeafEpsilon) < 0.0;
                    if (!S.leaf) {
                        const int32_t ps = int32_t(lo + pos), d = rec.depth + 1, id = int32_t(S.node_count);
                        const int32_t nc = int32_t(S.n_const_out);
                        T.stack[S.stack_top++] = StackRec{ps, int32_t(hi), d, id, 0, nc, gr};
                        T.stack[S.stack_top++] = StackRec{int32_t(lo), ps, d, id, 1, nc, gl};
                    }
                }
            }
            tm.sync();
        }
        if (tm.tid == 0) {
            const int64_t id = S.node_count++;
            NodeOut &o = T.nodes[id];
            o.n_samples = int32_t(m);
            o.impurity = S.imp;
            o.weighted = S.wn;
            o.pad = 0;
            if (S.leaf) {
                o.left = o.right = kTreeLeaf;
                o.feature = kTreeUndefined;
                o.threshold = double(kTreeUndefined);
                o.missing_left = 0;
            } else {
                o.left = o.right = 0;
                o.feature = S.best_f;
                o.threshold = S.best_thr;
                o.missing_left = S.best_missing_left;
            }
            if (rec.parent != kTreeUndefined) {
                if (rec.is_left) T.nodes[rec.parent].left = int32_t(id);
                else T.nodes[rec.parent].right = int32_t(id);
            }
            T.values[id] = ddiv(S.sum_total, S.wn);
            if (rec.depth > S.max_depth) S.max_depth = rec.depth;
        }
        tm.sync();
    }
}

// ------------------------------------------------------------------------------------------------
// Gradient boosting: GradientBoostingClassifier(n_estimators).fit with the library's arguments (loss="log_loss",
// learning_rate=0.1, max_depth=3, subsample=1.0), one stage's trees.  _fit_stage (ensemble/_gb.py) fits k = 0 .. K - 1
// DecisionTreeRegressor(squared_error, best splitter, max_depth=3, max_features=None) on column k of the stage's negative
// gradient with unit weights: build_regression_tree with max_depth 3, all-ones weights and y_stride K.  The gradient
// itself (exp / log) is computed on the host by scikit-learn's own loss object; everything here is ordered float64
// arithmetic.  _update_terminal_regions then replaces every leaf's value by one Newton step over the rows tree.apply puts
// in it, in ascending row order:
//   numerator   = np.average(neg_g, weights=1) = pairwise_sum(neg_g) / count, times (K - 1) / K for the multinomial loss
//   denominator = np.average(prob * (1 - prob), weights=1), prob = y_k - neg_g (y_k: y for the binomial loss, the
//                 one-hot column y == k for the multinomial one)
//   value       = 0.0 when |denominator| < 1e-150 (_safe_divide), else numerator / denominator
// and adds learning_rate * value[leaf] to raw[:, k].  Internal nodes keep the builder's mean.
constexpr int kBoostDepth = 3;                              // GradientBoostingClassifier's max_depth

// Dynamic shared memory of boost_build_kernel: the regression tree's and part [kThreads]; the attribute is set to
// kBoostSmemCap (as kSmemCap)
constexpr size_t boost_smem_bytes(int F) { return reg_smem_bytes(F) + size_t(kThreads) * 8; }
constexpr size_t kBoostSmemCap = boost_smem_bytes(kMaxFeats);

// One boosting tree's extras: its problem's class indices y [n] (0 / 1 for the binomial loss), the tree's raw column k of
// K, the training raw predictions raw [n, K], the learning rate, leaf_of / leaf_rows [n] (global) and part [team size].
struct BoostTree {
    const int32_t *y;
    int k, K;
    double *raw;
    double lr;
    int32_t *leaf_of, *leaf_rows;
    int64_t *part;
};

// tree.apply for one row: left iff x <= threshold (tree/_tree.pyx _apply_dense, float32 compared in float64)
template <class Xf>
__host__ __device__ inline int32_t tree_apply(const NodeOut *nodes, const Xf &x)
{
    int32_t i = 0;
    while (nodes[i].left != kTreeLeaf) i = double(x(nodes[i].feature)) <= nodes[i].threshold ? nodes[i].left : nodes[i].right;
    return i;
}

// np.add.reduce of a leaf's cnt terms: +0.0 plus NumPy's pairwise sum, without the recursion of npy::pairwise_sum (its
// frames are not in the kernel's static stack size)
template <class G>
__host__ __device__ inline double leaf_sum(const G &get, int64_t cnt)
{
    return front::np_sum(get, cnt, true);
}

// _safe_divide(numerator, denominator) of one leaf from its sums over cnt rows
__host__ __device__ inline double newton_value(double num_sum, double den_sum, int64_t cnt, int K)
{
    double num = ddiv(num_sum, double(cnt));
    if (K > 1) num = dmul(num, ddiv(double(K - 1), double(K)));
    const double den = ddiv(den_sum, double(cnt));
    return fabs(den) < 1e-150 ? 0.0 : ddiv(num, den);
}

// After build_regression_tree(T): every leaf's Newton value into T.values, then raw[:, k] += lr * value[leaf] for every
// training row.  Team-parallel but for the leaf sums (thread 0, one leaf after another).
__host__ __device__ inline void boost_leaves(const RegTree &T, const BoostTree &B, const Team &tm)
{
    const int64_t n = T.n;
    for (int64_t s = tm.tid; s < n; s += tm.n)
        B.leaf_of[s] = tree_apply(T.nodes, [&T, s](int f) { return T.x(int32_t(s), f); });
    tm.sync();
    const int64_t node_count = T.st->node_count, chunk = (n + tm.n - 1) / tm.n;
    const int64_t q0 = tm.tid * chunk, q1 = q0 + chunk < n ? q0 + chunk : n;
    for (int64_t id = 0; id < node_count; ++id) {
        if (T.nodes[id].left != kTreeLeaf) continue;
        // np.nonzero(masked_terminal_regions == leaf): the leaf's rows in ascending order, each thread's chunk after the
        // earlier chunks'
        int64_t c = 0;
        for (int64_t q = q0; q < q1; ++q) c += B.leaf_of[q] == id;
        B.part[tm.tid] = c;
        tm.sync();
        int64_t o = 0;
        for (int t = 0; t < tm.tid; ++t) o += B.part[t];
        for (int64_t q = q0; q < q1; ++q) {
            const int32_t s = int32_t(q);
            if (B.leaf_of[s] == id) B.leaf_rows[o++] = s;
        }
        tm.sync();
        if (tm.tid == 0) {
            int64_t cnt = 0;
            for (int t = 0; t < tm.n; ++t) cnt += B.part[t];
            const int32_t *rw = B.leaf_rows;
            const double num = leaf_sum([&T, rw](int64_t i) { return T.yv(rw[i]); }, cnt);
            const double den = leaf_sum([&T, &B, rw](int64_t i) {
                const int32_t s = rw[i];
                const double yk = B.K == 1 ? double(B.y[s]) : (B.y[s] == B.k ? 1.0 : 0.0);
                const double prob = dsub(yk, T.yv(s));
                return dmul(prob, dsub(1.0, prob));
            }, cnt);
            T.values[id] = newton_value(num, den, cnt, B.K);
        }
        tm.sync();
    }
    for (int64_t s = tm.tid; s < n; s += tm.n) {
        double &r = B.raw[s * B.K + B.k];
        r = dadd(r, dmul(B.lr, T.values[B.leaf_of[s]]));
    }
    tm.sync();
}

// predict's class of one row from its K raw scores (local class index): raw >= 0 for the binomial loss, else the first
// maximum (np.argmax)
__host__ __device__ inline int boost_class(const double *raw, int K)
{
    if (K == 1) return raw[0] >= 0.0 ? 1 : 0;
    int b = 0;
    for (int c = 1; c < K; ++c)
        if (raw[c] > raw[b]) b = c;
    return b;
}

}  // namespace forest
}  // namespace b200aa
