// Beat extraction (kernel 4): the per-row pieces of MidTermFeatures.beat_extraction (reference MidTermFeatures.py:18-84,
// peak picking from utilities.peakdet :33-103) in the order of double operations the host function performs, so the
// kernel's (bpm, ratio) equal the host's bit for bit.  __host__ __device__: tests/beat_host.cu runs the same code on the CPU.
//
// Every double operation goes through dadd / dsub / dmul / ddiv (npsum.cuh), the correctly rounded intrinsics on the device.
#pragma once
#include <cmath>
#include <cstdint>

#include "npsum.cuh"

namespace b200aa {
namespace beat {

constexpr int kRows = 18;               // _BEAT_ROWS: short-term rows 0, 1, 3 .. 18 (MidTermFeatures.py:31-32)
constexpr int kChunk = 1024;            // frames per chunk of the scan: shorter rows are a single chunk

__host__ __device__ inline int row_index(int r) { return r < 2 ? r : r + 1; }

using npy::dadd;
using npy::ddiv;
using npy::dmul;
using npy::dsub;
using npy::pairwise_part;
using npy::pairwise_sum;

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
