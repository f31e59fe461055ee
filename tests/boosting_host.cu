// Host program for tests/test_boosting_cpu.py: runs one gradient boosting stage of kernel 13 (pyaudioanalysis_b200/csrc/
// forest.cuh: build_regression_tree with max_depth 3, then boost_leaves) on the CPU, with a team of TEAM threads
// (tests/team_host.h; default 1).
//
//   boosting_host stage IN OUT [TEAM]
//                                  IN: int64 n, n_feats, K; float32 X [n, n_feats]; float64 neg_g [n, K]; int32 y [n];
//                                      float64 raw [n, K]; uint32 rand_r seeds [K]; float64 learning_rate
//                                  OUT: per tree k: int64 node_count, max_depth; nodes [node_count] (48-byte
//                                       forest::NodeOut); float64 values [node_count]; then float64 raw [n, K]
//   boosting_host predict IN OUT   IN: int64 n, K; float64 raw [n, K]    OUT: int32 boost_class of every row [n]
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
    if (!strcmp(argv[1], "predict")) {
        const std::vector<int64_t> h = rd<int64_t>(in, 2);
        const int K = int(h[1]);
        const std::vector<double> raw = rd<double>(in, size_t(h[0]) * K);
        for (int64_t i = 0; i < h[0]; ++i) {
            const int32_t c = forest::boost_class(raw.data() + i * K, K);
            fwrite(&c, 4, 1, out);
        }
        fclose(out);
        return 0;
    }
    const std::vector<int64_t> h = rd<int64_t>(in, 3);
    const int64_t n = h[0];
    const int F = int(h[1]), K = int(h[2]);
    const std::vector<float> X = rd<float>(in, size_t(n) * F);
    const std::vector<double> neg_g = rd<double>(in, size_t(n) * K);
    const std::vector<int32_t> y = rd<int32_t>(in, size_t(n));
    std::vector<double> raw = rd<double>(in, size_t(n) * K);
    const std::vector<uint32_t> seeds = rd<uint32_t>(in, size_t(K));
    const double lr = rd<double>(in, 1)[0];
    fclose(in);
    std::vector<int32_t> w(n, 1), samples(n), idx(n), features(F), constf(F), drawn(F), vis(F), tied(F), leaf_of(n), rows(n);
    std::vector<float> fv(n), mn(F), mx(F);
    std::vector<uint64_t> keys(size_t(F) * forest::pow2_at_least(n));
    std::vector<forest::StackRec> stack(n + 1);
    std::vector<forest::NodeOut> nodes(2 * n - 1);
    std::vector<double> values(2 * n - 1), vproxy(F);
    std::vector<int64_t> vpos(F), part(team);
    forest::RegShared st{};
    for (int k = 0; k < K; ++k) {
        const forest::RegTree T{X.data(), neg_g.data() + k, nullptr, w.data(), n, F, samples.data(), idx.data(), fv.data(),
                                keys.data(), stack.data(), nodes.data(), values.data(), features.data(), constf.data(),
                                drawn.data(), vis.data(), tied.data(), mn.data(), mx.data(), vproxy.data(), vpos.data(), &st,
                                K, forest::kBoostDepth};
        const forest::BoostTree B{y.data(), k, K, raw.data(), lr, leaf_of.data(), rows.data(), part.data()};
        team_host::run_team(team, [&](const forest::Team &tm) {
            forest::build_regression_tree(T, tm, seeds[k]);
            forest::boost_leaves(T, B, tm);
        });
        const int64_t head[2] = {st.node_count, st.max_depth};
        fwrite(head, sizeof(int64_t), 2, out);
        fwrite(nodes.data(), sizeof(forest::NodeOut), size_t(st.node_count), out);
        fwrite(values.data(), sizeof(double), size_t(st.node_count), out);
    }
    fwrite(raw.data(), sizeof(double), raw.size(), out);
    fclose(out);
    return 0;
}
