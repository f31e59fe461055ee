// Work distribution of the warp-autonomous kernels (pair_kernel.cuh, solo_kernel.cuh): static shares + steal-half.
//
// The launch's pair steps form one sequence g in [0, total), g = clip * pairs_per_clip + q.  Warp w starts with the
// contiguous share [w total / W, (w + 1) total / W) and takes it from the front, `chunk` pairs per atomic; a warp that runs
// dry takes the BACK half of the largest remainder it finds among 256 descriptors at a time and goes on from there.  A
// contiguous run needs the one-pair halo (flux and the deltas look one frame back) only where it starts, so the redundant
// work is one pair step per warp and per steal.  What it took to get there (DESIGN.md): the scans
// below must be cheap (the first version's last-warp scans cost more than the halos saved) and every branch must hang on a
// vote, or ptxas stops trusting the warp's convergence in the step loop that follows.
//
// State: one 64-bit word per warp, (back << 32) | front, 0 = its warp has not started yet (a memset is all a launch needs;
// nobody steals from a warp that has not started, and no warp ever waits for another: correctness does not rest on all CTAs
// being resident at once -- beside another stream's kernels some start only when others have finished); every
// transition is a single atomic on that word: the owner's claim is an atomicAdd on the front half, a steal is a
// compare-and-swap that lowers the back half (it fails, harmlessly, if the owner moved in between), and a thief publishes
// what it took with an atomicExch on its own word.  The functions are host + device so that tests/sched_host.cpp can run
// them with one CPU thread per "warp" (tests/test_sched_cpu.py).  The nvcc-only part below also holds the host side of a
// launch that the persistent kernels' launchers share: the steal-schedule setup and the resident-CTA count.
#pragma once
#include <cstdint>
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include "../../include/b200aa.h"
#define B200AA_HD __host__ __device__ __forceinline__
#else
#define B200AA_HD inline
#endif

namespace b200aa {

struct StealParams {
    unsigned long long *ranges;     // [n_warps], zeroed in-stream before the launch
    unsigned n_warps;               // gridDim.x * warps per CTA
    unsigned total;                 // pair steps of the launch (< 2^31)
    unsigned per_clip;              // pair steps per (full-length) clip
    unsigned chunk;                 // pairs per claim
    unsigned min_steal;             // smallest remainder worth splitting (>= 2: a steal takes half, rounded down)
};

B200AA_HD unsigned long long sched_pack(unsigned front, unsigned back) { return (static_cast<unsigned long long>(back) << 32) | front; }

B200AA_HD void sched_initial(const StealParams &sp, unsigned w, unsigned &front, unsigned &back)
{
    front = static_cast<unsigned>(static_cast<unsigned long long>(w) * sp.total / sp.n_warps);
    back = static_cast<unsigned>(static_cast<unsigned long long>(w + 1) * sp.total / sp.n_warps);
}

B200AA_HD void sched_decode(unsigned long long raw, unsigned &front, unsigned &back)
{
    front = static_cast<unsigned>(raw & 0xffffffffull);         // (0 decodes to the empty range)
    back = static_cast<unsigned>(raw >> 32);
}

// ---- the three atomics (device: CUDA atomics on global memory; host: GCC builtins, for the CPU test)
B200AA_HD unsigned long long sched_add(unsigned long long *p, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST);
#endif
}
B200AA_HD unsigned long long sched_cas(unsigned long long *p, unsigned long long expect, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, expect, v);
#else
    __atomic_compare_exchange_n(p, &expect, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return expect;          // the value found (== the expected one on success)
#endif
}
B200AA_HD void sched_store(unsigned long long *p, unsigned long long v)
{
#if defined(__CUDA_ARCH__)
    atomicExch(p, v);
#else
    __atomic_store_n(p, v, __ATOMIC_SEQ_CST);
#endif
}
B200AA_HD unsigned long long sched_load(const unsigned long long *p)
{
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const volatile unsigned long long *>(p);
#else
    return __atomic_load_n(p, __ATOMIC_SEQ_CST);
#endif
}

// owner, once: publish the initial share
B200AA_HD void sched_begin(const StealParams &sp, unsigned w)
{
    unsigned f, b;
    sched_initial(sp, w, f, b);
    sched_store(sp.ranges + w, sched_pack(f, b));
}

// owner: the next `inc` pairs of the own range; false = nothing left.  `inc` is then set for the next claim: a quarter of
// what is left, between 1 and sp.chunk -- claimed pairs cannot be stolen any more, so the claims shrink towards the end of
// the range and the last pairs of a launch change hands one at a time (the tail of the kernel is one or two pair steps).
B200AA_HD bool sched_claim(const StealParams &sp, unsigned w, unsigned &inc, unsigned &g0, unsigned &g1)
{
    const unsigned long long old = sched_add(sp.ranges + w, static_cast<unsigned long long>(inc));
    unsigned f, b;
    sched_decode(old, f, b);
    if (f >= b) return false;
    g0 = f;
    g1 = (b - f < inc) ? b : f + inc;
    const unsigned q = (b - g1) / 4u;
    inc = q < 1u ? 1u : (q > sp.chunk ? sp.chunk : q);
    return true;
}

// remainder of descriptor v as read (`raw`); 0 if it is not worth splitting
B200AA_HD unsigned sched_remainder(const StealParams &sp, unsigned long long raw)
{
    unsigned f, b;
    sched_decode(raw, f, b);
    if (b <= f) return 0u;
    const unsigned rem = b - f;
    return rem >= sp.min_steal ? rem : 0u;
}

// thief w: take the back half of victim v's remainder (as read in `raw`) and publish it as the own range
B200AA_HD bool sched_try_steal(const StealParams &sp, unsigned w, unsigned v, unsigned long long raw)
{
    unsigned f, b;
    sched_decode(raw, f, b);
    if (b <= f || b - f < sp.min_steal) return false;
    const unsigned take = (b - f) / 2;
    const unsigned nb = b - take;
    if (sched_cas(sp.ranges + v, raw, sched_pack(f, nb)) != raw) return false;
    sched_store(sp.ranges + w, sched_pack(nb, b));
    return true;
}

#if defined(__CUDACC__)
// thief (whole warp): scan the descriptors 256 at a time (eight independent loads per lane in flight: a scan of 3 000 words
// is a dozen L2 round trips -- one dependent load per 32 words made the last warps' scans the kernel's tail) from a
// warp-specific offset and split the largest remainder of the first window that has one;
// false = nothing worth taking anywhere (the warp is done).
// Every decision is taken on a vote / reduction result, so the warp provably stays converged.
__device__ __forceinline__ bool sched_steal(const StealParams &sp, unsigned w, int lane)
{
    constexpr int U = 8;
    const unsigned n = sp.n_warps;
    const unsigned start = (w * 977u + 131u) % n;
    for (int attempt = 0; attempt < 2; ++attempt) {
        bool contended = false;
        for (unsigned off = 0; off < n; off += 32 * U) {
            unsigned long long raw[U];
            unsigned idx[U];
#pragma unroll
            for (int j = 0; j < U; ++j) {
                const unsigned o = off + unsigned(j) * 32u + unsigned(lane);
                const unsigned i = start + o;               // start < n: one conditional subtraction wraps it
                idx[j] = o < n ? (i >= n ? i - n : i) : w;  // out of range: skipped like the own word
                raw[j] = o < n ? sched_load(sp.ranges + idx[j]) : 0ull;
            }
            unsigned best = 0u, bv = w;
            unsigned long long braw = 0ull;
#pragma unroll
            for (int j = 0; j < U; ++j) {
                const unsigned rem = idx[j] != w ? sched_remainder(sp, raw[j]) : 0u;
                if (rem > best) { best = rem; bv = idx[j]; braw = raw[j]; }
            }
            const unsigned wbest = __reduce_max_sync(0xffffffffu, best);
            if (wbest == 0u) continue;
            const unsigned holders = __ballot_sync(0xffffffffu, best == wbest);
            const int bl = __ffs(int(holders)) - 1;
            const bool mine = lane == bl && sched_try_steal(sp, w, bv, braw);
            if (__any_sync(0xffffffffu, mine)) return true;
            contended = true;               // somebody else got there first
        }
        if (!contended) break;
    }
    return false;
}

// whole warp: next chunk [g0, g1) of the launch.  1 = a chunk of the own range; 2 = the own range was empty and a steal
// refilled it (call again); 0 = the warp is done.  (One claim per call, no loop in here: with a claim-or-steal loop inside,
// ptxas no longer proves the warp converged at the kernels' step loops and wraps each of their shuffles in WARPSYNC /
// ENDCOLLECTIVE sequences -- measured: 330 of them, +3 % instructions, 50 more spilled words.)
__device__ __forceinline__ int sched_next(const StealParams &sp, unsigned w, int lane, unsigned &inc, unsigned &g0, unsigned &g1)
{
    unsigned a = 0, b = 0, ni = inc;
    bool got = false;
    if (lane == 0) got = sched_claim(sp, w, ni, a, b);
    if (__any_sync(0xffffffffu, got)) {
        g0 = __shfl_sync(0xffffffffu, a, 0);
        g1 = __shfl_sync(0xffffffffu, b, 0);
        inc = __shfl_sync(0xffffffffu, ni, 0);
        return 1;
    }
    inc = 1u;                           // a stolen range starts with a single pair (it is small near the end of a launch)
    return sched_steal(sp, w, lane) ? 2 : 0;
}

// ---- host side of a launch
// Steal schedule of one launch of `total` pair steps (per_clip per clip) in CTAs of `warps` warps: small launches shrink
// `grid` to as many warps as they have pairs, every warp gets a range descriptor in `ranges` (ranges_cap bytes), zeroed
// in-stream.  B200AA_PAIR_STEAL="chunk,min_steal" overrides the claim size and the smallest remainder worth splitting
// (tuning).  B200AA_ERR_UNSUPPORTED: the launch does not fit 32-bit steps or the descriptors do not fit `ranges`.
inline int steal_setup(StealParams &sp, unsigned long long *ranges, size_t ranges_cap, int64_t total, int64_t per_clip,
                       int warps, int64_t &grid, cudaStream_t st)
{
    if (total >= (int64_t(1) << 31)) return B200AA_ERR_UNSUPPORTED;
    if (grid * warps > total) grid = (total + warps - 1) / warps;
    const int64_t n_warps = grid * warps;
    if (size_t(n_warps) * sizeof(unsigned long long) > ranges_cap) return B200AA_ERR_UNSUPPORTED;
    long chunk = 8, min_steal = 2;
    if (const char *ov = getenv("B200AA_PAIR_STEAL")) {
        long a = 0, b2 = 0;
        if (sscanf(ov, "%ld,%ld", &a, &b2) == 2 && a > 0 && a <= 65536 && b2 > 1 && b2 <= 65536) { chunk = a; min_steal = b2; }
    }
    sp.ranges = ranges;
    sp.n_warps = unsigned(n_warps);
    sp.total = unsigned(total);
    sp.per_clip = unsigned(per_clip);
    sp.chunk = unsigned(chunk);
    sp.min_steal = unsigned(min_steal);
    if (cudaMemsetAsync(ranges, 0, size_t(n_warps) * sizeof(unsigned long long), st) != cudaSuccess) return B200AA_ERR_CUDA;
    return B200AA_OK;
}

// Resident CTAs per SM of `kern` at `threads` threads and `smem` dynamic shared bytes, at least 1.  The kernel's shared-memory
// cap is always set to the launcher's constant `cap`, so concurrent launches of one instantiation cannot undercut each other.
template <class Kernel>
inline cudaError_t resident_ctas(Kernel kern, int threads, size_t smem, int cap, int &occ)
{
    occ = 1;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem);
    if (occ < 1) occ = 1;
    return e;
}
#endif

}  // namespace b200aa
