// Beat extraction (kernel 4): the per-row pieces of MidTermFeatures.beat_extraction (reference MidTermFeatures.py:18-84,
// peak picking from utilities.peakdet :33-103) in the order of double operations the host function performs, so the
// kernel's (bpm, ratio) equal the host's bit for bit.  __host__ __device__: tests/beat_host.cu runs the same code on the CPU.
//
// Every double operation goes through dadd / dsub / dmul / ddiv, which are the correctly rounded intrinsics on the device:
// no FMA contraction, and no division expanded into an FMA sequence.
#pragma once
#include <cmath>
#include <cstdint>

namespace b200aa {
namespace beat {

constexpr int kRows = 18;               // _BEAT_ROWS: short-term rows 0, 1, 3 .. 18 (MidTermFeatures.py:31-32)
constexpr int kChunk = 1024;            // frames per chunk of the scan: shorter rows are a single chunk
constexpr int kLeaf = 128;              // NumPy's PW_BLOCKSIZE

__host__ __device__ inline int row_index(int r) { return r < 2 ? r : r + 1; }

__host__ __device__ inline double dadd(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline double dsub(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline double dmul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline double ddiv(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// np.add.reduce of get(off) .. get(off + n - 1): NumPy's pairwise summation.  Below 8 elements a running sum from 0.0; up to
// 128, eight running accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added in sequence; above 128,
// a split at n/2 rounded down to a multiple of 8.  Elements at index >= nz are +0.0 and are not read: the sums here are of
// values >= +0.0 (or NaN), for which x + 0.0 == x, so a subtree lying entirely at or beyond nz sums to +0.0 whatever its shape.
template <class G>
__host__ __device__ double pairwise_sum(const G &get, int64_t off, int64_t n, int64_t nz)
{
    if (n <= 0 || off >= nz) return 0.0;
    auto at = [&](int64_t i) { return i < nz ? get(i) : 0.0; };
    if (n < 8) {
        double r = 0.0;
        for (int64_t i = 0; i < n; ++i) r = dadd(r, at(off + i));
        return r;
    }
    if (n <= kLeaf) {
        double r[8];
        for (int j = 0; j < 8; ++j) r[j] = at(off + j);
        int64_t i = 8;
        for (; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; ++j) r[j] = dadd(r[j], at(off + i + j));
        double res = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
        for (; i < n; ++i) res = dadd(res, at(off + i));
        return res;
    }
    int64_t n2 = n / 2;
    n2 -= n2 % 8;
    return dadd(pairwise_sum(get, off, n2, nz), pairwise_sum(get, off + n2, n - n2, nz));
}

// The subtree of pairwise_sum(n) that lane k of 2^levels lanes sums: `levels` splits, taken along k's bits from the top.  A leaf
// reached early stays with the leftmost lane below it; the other lanes get an empty range.  Combining the lane sums as
// s[k] = s[k] + s[k + 2^j] for j = 0 .. levels - 1 (k a multiple of 2^(j+1)) then reproduces the tree: a split node adds its
// halves left + right, and a leaf adds only +0.0s.
__host__ __device__ inline void pairwise_part(int64_t n, int levels, int k, int64_t &off, int64_t &len)
{
    off = 0;
    len = n;
    for (int j = levels - 1; j >= 0; --j) {
        const int bit = (k >> j) & 1;
        if (len > kLeaf) {
            int64_t n2 = len / 2;
            n2 -= n2 % 8;
            if (bit) { off += n2; len -= n2; } else { len = n2; }
        } else if (bit) {
            len = 0;
        }
    }
}

// thr = 2 * mean(|row[:-1] - row[1:]|) from the pairwise sum of the T - 1 differences (NaN for T <= 1, the mean of an empty
// slice); a threshold <= 0 becomes 1e-16 (MidTermFeatures.py:36-39)
__host__ __device__ inline double threshold(double sum, int64_t T)
{
    const int64_t n = T > 1 ? T - 1 : 0;
    double thr = dmul(2.0, ddiv(sum, double(n)));
    if (thr <= 0) thr = 0.0000000000000001;
    return thr;
}

// State of peakdet's scan.  After a switch to "look for min" mx / mxpos are dead until the next switch overwrites them; after a
// switch to "look for max" mn is dead.  So two scans whose live parts agree after the same index emit the same peaks from
// then on.
struct State {
    double mx, mn;
    int32_t mxpos, lfm;
};

__host__ __device__ inline State fresh() { return State{-INFINITY, INFINITY, 0, 1}; }

// one step of peakdet at index i (strict comparisons; NaN fails all of them): the emitted peak's position, or -1
__host__ __device__ inline int32_t step(State &s, double x, int32_t i, double delta)
{
    if (x > s.mx) { s.mx = x; s.mxpos = i; }
    if (x < s.mn) s.mn = x;
    if (s.lfm) {
        if (x < dsub(s.mx, delta)) { s.mn = x; s.lfm = 0; return s.mxpos; }
    } else if (x > dadd(s.mn, delta)) {
        s.mx = x; s.mxpos = i; s.lfm = 1;
    }
    return -1;
}

__host__ __device__ inline bool same_future(const State &a, const State &b)
{
    return a.lfm == b.lfm && (a.lfm ? (a.mx == b.mx && a.mxpos == b.mxpos) : a.mn == b.mn);
}

// One chunk [c0, c1) of a row.  After the speculative pass: the exit state of a scan started fresh at c0, its last emitted peak
// and the index at which it was emitted (-1: none).  After the fix-up: the true entry state and the last peak before c0.
struct Chunk {
    State s;
    int32_t last, last_at;
};

template <class V>
__host__ __device__ Chunk spec_chunk(const V &v, int32_t c0, int32_t c1, double delta)
{
    Chunk r{fresh(), -1, -1};
    for (int32_t i = c0; i < c1; ++i) {
        const int32_t p = step(r.s, v(i), i, delta);
        if (p >= 0) { r.last = p; r.last_at = i; }
    }
    return r;
}

// Fix-up of one chunk: `s` / `last` enter as the true state and last peak at c0 and leave as those at c1.  The true scan and a
// fresh one run side by side until their live states agree; from there on the speculative record holds the rest of the chunk.
// A chunk where they never agree is scanned to its end, so the worst case is the serial scan.
template <class V>
__host__ __device__ void fixup_chunk(const V &v, int32_t c0, int32_t c1, double delta, const Chunk &spec, State &s, int32_t &last)
{
    State t = fresh();
    for (int32_t i = c0; i < c1; ++i) {
        const double x = v(i);
        const int32_t p = step(s, x, i, delta);
        if (p >= 0) last = p;
        step(t, x, i, delta);
        if (same_future(s, t)) {
            s = spec.s;
            if (spec.last_at > i) last = spec.last;
            return;
        }
    }
}

// scan [c0, c1) from state s, calling emit(p) for every peak
template <class V, class E>
__host__ __device__ void scan_chunk(const V &v, int32_t c0, int32_t c1, double delta, State s, const E &emit)
{
    for (int32_t i = c0; i < c1; ++i) {
        const int32_t p = step(s, v(i), i, delta);
        if (p >= 0) emit(p);
    }
}

}  // namespace beat
}  // namespace b200aa
