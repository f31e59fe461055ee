// Host program for tests/test_knn_cpu.py: runs the __host__ __device__ pieces of kernel 5 (pyaudioanalysis_b200/csrc/knn.cuh)
// on the CPU in the order the kernels apply them.  Reads commands from stdin, numbers as C hex floats / "inf" / "nan";
// prints results as hex floats ("nan" for NaN) and keys as hex integers.
//
//   dist N F n  v (N x F)  x (n x F)                 -> per query: its n distances to the N training rows
//   key m d_1 .. d_m                                 -> the m sort keys
//   classify N F C k  slots (N)  v (N x F)  n  x (n x F) -> per query: the id and the C votes
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../pyaudioanalysis_b200/csrc/knn.cuh"
#include "host_io.h"

using namespace b200aa;

// the select kernel for one query: radix select of the k-th smallest key, the ordered pass, the votes and the first maximum
static void classify(const std::vector<uint64_t> &keys, const std::vector<int> &slots, int C, int64_t k)
{
    const int64_t N = int64_t(keys.size());
    uint64_t thr = knn::kAll;
    int64_t r = 0;
    if (k < N) {
        uint64_t prefix = 0;
        int64_t rank = k;
        for (int shift = 64 - knn::kDigitBits; shift >= 0; shift -= knn::kDigitBits) {
            const uint64_t mask = knn::prefix_mask(shift);
            unsigned hist[knn::kBins] = {};
            for (int64_t i = 0; i < N; ++i)
                if ((keys[i] & mask) == prefix) hist[(keys[i] >> shift) & (knn::kBins - 1)]++;
            prefix |= uint64_t(knn::select_digit(hist, rank)) << shift;
        }
        thr = prefix;
        r = rank;
    }
    std::vector<int64_t> votes(C, 0);
    int64_t equal_before = 0;
    for (int64_t i = 0; i < N; ++i) {
        if (knn::selected(keys[i], thr, equal_before, r) && slots[i] >= 0 && slots[i] < C) votes[slots[i]]++;
        if (keys[i] == thr) ++equal_before;
    }
    int64_t bc = -1, bi = 0;
    for (int c = 0; c < C; ++c)
        if (bc < 0 || knn::better(votes[c], c, bc, bi)) { bc = votes[c]; bi = c; }
    printf("classify %lld", (long long)bi);
    for (int c = 0; c < C; ++c) pr(knn::vote(votes[c], k));
    printf("\n");
}

int main()
{
    char cmd[16];
    while (scanf("%15s", cmd) == 1) {
        if (!strcmp(cmd, "dist")) {
            const int64_t N = rl();
            const int F = int(rl());
            const int64_t n = rl();
            const std::vector<double> v = rv(size_t(N) * F), x = rv(size_t(n) * F);
            for (int64_t q = 0; q < n; ++q) {
                printf("dist");
                for (int64_t i = 0; i < N; ++i)
                    pr(knn::distance([&](int j) { return x[size_t(q) * F + j]; }, [&](int j) { return v[size_t(i) * F + j]; }, F));
                printf("\n");
            }
        } else if (!strcmp(cmd, "key")) {
            const int64_t m = rl();
            printf("key");
            for (int64_t i = 0; i < m; ++i) printf(" %llx", (unsigned long long)knn::key_of(rd()));
            printf("\n");
        } else if (!strcmp(cmd, "classify")) {
            const int64_t N = rl();
            const int F = int(rl()), C = int(rl());
            const int64_t k = rl();
            std::vector<int> slots(N);
            for (auto &s : slots) s = int(rl());
            const std::vector<double> v = rv(size_t(N) * F);
            const int64_t n = rl();
            const std::vector<double> x = rv(size_t(n) * F);
            std::vector<uint64_t> keys(N);
            for (int64_t q = 0; q < n; ++q) {
                for (int64_t i = 0; i < N; ++i)
                    keys[i] = knn::key_of(
                        knn::distance([&](int j) { return x[size_t(q) * F + j]; }, [&](int j) { return v[size_t(i) * F + j]; }, F));
                classify(keys, slots, C, k);
            }
        } else {
            return 2;
        }
    }
    return 0;
}
