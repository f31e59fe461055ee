// Host program for tests/test_trees_cpu.py: runs the __host__ __device__ pieces of kernel 8
// (pyaudioanalysis_b200/csrc/trees.cuh) on the CPU, one row at a time, in the order the kernel applies them: the float32
// cast and refusal flag, the walk of every tree, each class's sum over the trees in tree order, the score and the id.
//
//   trees_host IN OUT
//   IN:  int64 n_nodes, n_trees, n_leaves, mode, n_classes, n_feats, allow_nan, dtype (1 float32, 2 float64), n_rows,
//        has_init; int32 nodes [n_nodes, 4]; int32 roots [n_trees]; float64 values [n_leaves, n_classes] (mode 0) or
//        [n_leaves] (mode 1); float64 init [n_classes] if has_init; queries [n_rows, n_feats] of the dtype
//   OUT: int64 ids [n_rows]; int32 bad [n_rows]; float64 scores [n_rows, n_classes]
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/trees.cuh"

using namespace b200aa;

template <class T>
static std::vector<T> rd(FILE *f, size_t n)
{
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) exit(3);
    return v;
}

template <class T>
static void classify(const std::vector<trees::Node> &nodes, const std::vector<int32_t> &roots, const std::vector<double> &values,
                     const std::vector<double> &init, int mode, int C, int F, bool allow_nan, const std::vector<T> &q,
                     int64_t n, std::vector<int64_t> &ids, std::vector<int32_t> &bad, std::vector<double> &scores)
{
    const int T_ = int(roots.size());
    std::vector<float> x(F);
    std::vector<double> acc(C);
    for (int64_t r = 0; r < n; ++r) {
        bool b = false;
        for (int j = 0; j < F; ++j) x[j] = trees::cast(q[size_t(r) * F + j], allow_nan, b);
        for (int c = 0; c < C; ++c) acc[c] = init.empty() ? 0.0 : init[c];
        for (int t = 0; t < T_; ++t) {
            const int32_t leaf = trees::walk(nodes.data(), roots[t], x.data());
            const int tc = trees::tree_class(mode, t, C);
            for (int c = 0; c < C; ++c) {
                if (tc < 0) acc[c] = trees::dadd(acc[c], values[size_t(leaf) * C + c]);
                else if (tc == c) acc[c] = trees::dadd(acc[c], values[leaf]);
            }
        }
        double best = 0.0;
        int bi = -1;
        for (int c = 0; c < C; ++c) {
            const double s = trees::finish(mode, acc[c], T_);
            scores[size_t(r) * C + c] = s;
            if (bi < 0 || trees::better(s, c, best, bi)) { best = s; bi = c; }
        }
        ids[r] = trees::class_id(mode, C, scores[size_t(r) * C], bi);
        bad[r] = b ? 1 : 0;
    }
}

int main(int argc, char **argv)
{
    if (argc != 3) return 2;
    FILE *in = fopen(argv[1], "rb");
    if (!in) return 2;
    const std::vector<int64_t> h = rd<int64_t>(in, 10);
    const int64_t n_nodes = h[0], n_trees = h[1], n_leaves = h[2], n = h[8];
    const int mode = int(h[3]), C = int(h[4]), F = int(h[5]);
    const bool allow_nan = h[6] != 0;
    const std::vector<trees::Node> nodes = rd<trees::Node>(in, size_t(n_nodes));
    const std::vector<int32_t> roots = rd<int32_t>(in, size_t(n_trees));
    const std::vector<double> values = rd<double>(in, size_t(n_leaves) * (mode == trees::kForestMean ? C : 1));
    const std::vector<double> init = rd<double>(in, h[9] ? size_t(C) : 0);
    std::vector<int64_t> ids(n);
    std::vector<int32_t> bad(n);
    std::vector<double> scores(size_t(n) * C);
    if (h[7] == 1) classify(nodes, roots, values, init, mode, C, F, allow_nan, rd<float>(in, size_t(n) * F), n, ids, bad, scores);
    else classify(nodes, roots, values, init, mode, C, F, allow_nan, rd<double>(in, size_t(n) * F), n, ids, bad, scores);
    fclose(in);
    FILE *out = fopen(argv[2], "wb");
    if (!out) return 2;
    fwrite(ids.data(), sizeof(int64_t), ids.size(), out);
    fwrite(bad.data(), sizeof(int32_t), bad.size(), out);
    fwrite(scores.data(), sizeof(double), scores.size(), out);
    fclose(out);
    return 0;
}
