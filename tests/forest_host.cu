// Host program for tests/test_forest_cpu.py: runs kernel 13's tree builder (pyaudioanalysis_b200/csrc/forest.cuh,
// build_tree) on the CPU with a team of TEAM threads (tests/team_host.h; default 1), tree after tree, over the same per-tree
// inputs the device kernel gets.
//
//   forest_host IN OUT [TEAM]
//   IN:  int64 n, n_feats, n_classes, kind, n_trees, max_features, has_weights; float32 X [n, n_feats]; int32 y [n];
//        int32 weights [n_trees, n] if has_weights; uint32 rand_r seeds [n_trees]
//   OUT: per tree: int64 node_count, max_depth; nodes [node_count] (48-byte forest::NodeOut); float64 values
//        [node_count, n_classes]
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "forest.cuh"
#include "team_host.h"

using namespace b200aa;

template <class T>
static std::vector<T> rd(FILE *f, size_t n)
{
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) exit(3);
    return v;
}

int main(int argc, char **argv)
{
    if (argc != 3 && argc != 4) return 2;
    const int team = argc == 4 ? atoi(argv[3]) : 1;
    if (team < 1 || team > forest::kThreads) return 2;
    FILE *in = fopen(argv[1], "rb");
    if (!in) return 2;
    const std::vector<int64_t> h = rd<int64_t>(in, 7);
    const int64_t n = h[0], n_trees = h[4];
    const int F = int(h[1]), C = int(h[2]), kind = int(h[3]), max_features = int(h[5]);
    const std::vector<float> X = rd<float>(in, size_t(n) * F);
    const std::vector<int32_t> y = rd<int32_t>(in, size_t(n));
    const std::vector<int32_t> w = rd<int32_t>(in, h[6] ? size_t(n_trees * n) : 0);
    const std::vector<uint32_t> seeds = rd<uint32_t>(in, size_t(n_trees));
    fclose(in);
    FILE *out = fopen(argv[2], "wb");
    if (!out) return 2;
    std::vector<int32_t> samples(n), tmp(n), features(F), constf(F), drawn(F);
    std::vector<uint64_t> keys(forest::pow2_at_least(n));
    std::vector<forest::StackRec> stack(n + 1);
    std::vector<forest::NodeOut> nodes(2 * n - 1);
    std::vector<double> values((2 * n - 1) * C), thr(F), red_proxy(team);
    std::vector<float> mn(F), mx(F);
    std::vector<int64_t> cnt(size_t(team) * C), red_pos(team);
    forest::Shared st{};
    for (int64_t t = 0; t < n_trees; ++t) {
        forest::Tree T{X.data(), y.data(), w.empty() ? nullptr : w.data() + t * n, n, F, C, max_features, kind,
                       samples.data(), tmp.data(), keys.data(), stack.data(), nodes.data(), values.data(),
                       features.data(), constf.data(), drawn.data(), mn.data(), mx.data(), thr.data(), cnt.data(),
                       red_proxy.data(), red_pos.data(), &st};
        team_host::run_team(team, [&](const forest::Team &tm) { forest::build_tree(T, tm, seeds[t]); });
        const int64_t head[2] = {st.node_count, st.max_depth};
        fwrite(head, sizeof(int64_t), 2, out);
        fwrite(nodes.data(), sizeof(forest::NodeOut), size_t(st.node_count), out);
        fwrite(values.data(), sizeof(double), size_t(st.node_count) * C, out);
    }
    fclose(out);
    return 0;
}
