// Host program for tests/test_forest_regression_cpu.py: runs kernel 13's regression pieces (pyaudioanalysis_b200/csrc/
// forest.cuh) on the CPU, with a team of TEAM threads for the tree builder (tests/team_host.h; default 1).
//
//   forest_regression_host sort IN OUT   IN: int64 n; float32 values [n]; int32 indices [n]
//                                        OUT: the values and indices after introsort_3way
//   forest_regression_host fit IN OUT [TEAM]
//                                        IN: int64 n, n_feats, n_trees; float32 X [n, n_feats]; float64 y [n];
//                                            int32 weights [n_trees, n]; uint32 rand_r seeds [n_trees]
//                                        OUT: per tree: int64 node_count, max_depth; nodes [node_count] (48-byte
//                                             forest::NodeOut); float64 values [node_count]
#include <cstdio>
#include <cstdlib>
#include <cstring>
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
    if (argc != 4 && argc != 5) return 2;
    const int team = argc == 5 ? atoi(argv[4]) : 1;
    if (team < 1 || team > forest::kThreads) return 2;
    FILE *in = fopen(argv[2], "rb");
    FILE *out = fopen(argv[3], "wb");
    if (!in || !out) return 2;
    if (!strcmp(argv[1], "sort")) {
        const int64_t n = rd<int64_t>(in, 1)[0];
        std::vector<float> v = rd<float>(in, size_t(n));
        std::vector<int32_t> ix = rd<int32_t>(in, size_t(n));
        forest::introsort_3way(v.data(), ix.data(), n);
        fwrite(v.data(), 4, size_t(n), out);
        fwrite(ix.data(), 4, size_t(n), out);
        fclose(out);
        return 0;
    }
    const std::vector<int64_t> h = rd<int64_t>(in, 3);
    const int64_t n = h[0], n_trees = h[2];
    const int F = int(h[1]);
    const std::vector<float> X = rd<float>(in, size_t(n) * F);
    const std::vector<double> y = rd<double>(in, size_t(n));
    const std::vector<int32_t> w = rd<int32_t>(in, size_t(n_trees * n));
    const std::vector<uint32_t> seeds = rd<uint32_t>(in, size_t(n_trees));
    fclose(in);
    std::vector<int32_t> samples(n), idx(n), features(F), constf(F), drawn(F), vis(F), tied(F);
    std::vector<float> fv(n), mn(F), mx(F);
    std::vector<uint64_t> keys(size_t(F) * forest::pow2_at_least(n));
    std::vector<forest::StackRec> stack(n + 1);
    std::vector<forest::NodeOut> nodes(2 * n - 1);
    std::vector<double> values(2 * n - 1), vproxy(F);
    std::vector<int64_t> vpos(F);
    forest::RegShared st{};
    for (int64_t t = 0; t < n_trees; ++t) {
        const forest::RegTree T{X.data(), y.data(), nullptr, w.data() + t * n, n, F, samples.data(), idx.data(), fv.data(),
                                keys.data(), stack.data(), nodes.data(), values.data(), features.data(), constf.data(),
                                drawn.data(), vis.data(), tied.data(), mn.data(), mx.data(), vproxy.data(), vpos.data(), &st};
        team_host::run_team(team, [&](const forest::Team &tm) { forest::build_regression_tree(T, tm, seeds[t]); });
        const int64_t head[2] = {st.node_count, st.max_depth};
        fwrite(head, sizeof(int64_t), 2, out);
        fwrite(nodes.data(), sizeof(forest::NodeOut), size_t(st.node_count), out);
        fwrite(values.data(), sizeof(double), size_t(st.node_count), out);
    }
    fclose(out);
    return 0;
}
