// libb200aa.so -- music thumbnails (kernel 10).
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/b200aa.h"
#include "entry.h"
#include "thumb.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 10: music_thumbnailing's self-similarity matrix, diagonal filter, masked argmax and walk (audioSegmentation.py:40-55,
// :1093-1180), bit for bit scipy and NumPy (csrc/thumb.cuh)
// ------------------------------------------------------------------------------------------------
// nrm[r] = sqrt(dot(x_r, x_r)) for every row of X
__global__ void __launch_bounds__(256) thumb_norm_kernel(const double *__restrict__ X, int64_t x_stride, int F, int64_t n,
                                                         double *__restrict__ nrm)
{
    for (int64_t r = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; r < n; r += int64_t(gridDim.x) * blockDim.x) {
        const double *x = X + r * x_stride;
        nrm[r] = npy::dsqrt(thumb::dot([x](int k) { return npy::dmul(x[k], x[k]); }, F));
    }
}

// One 64 x 64 tile of a track's S per CTA, upper-triangle tiles only (blockIdx.y: the track, blockIdx.x strides over its
// tiles).  Both sides are staged kF features at a time, as [feature][frame]; each thread runs 4 x 4 dot products (frames
// ty + 16a against tx + 16b), each with scipy's even and odd accumulators.  An odd F's last feature is still staged after
// the loop and added last.  Every entry is written twice, at (u, v) and (v, u); a NaN sets the track's flag.
__global__ void __launch_bounds__(thumb::kThreads, 2) thumb_sim_kernel(const thumb::Track *__restrict__ tracks,
                                                                      const double *__restrict__ X, int64_t x_stride, int F,
                                                                      const double *__restrict__ nrm,
                                                                      double *__restrict__ S, int32_t *__restrict__ nan_flag)
{
    using namespace thumb;
    __shared__ double sl[kF][kTile + 1];
    __shared__ double sr[kF][kTile + 1];
    const Track tr = tracks[blockIdx.y];
    const int64_t nt = (tr.T + kTile - 1) / kTile;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const double *Xt = X + tr.x0 * x_stride;
    double *St = S + tr.s0;
    for (int64_t l = blockIdx.x; l < upper_tiles(nt); l += gridDim.x) {
        int64_t ti, tj;
        upper_tile(l, nt, ti, tj);
        const int64_t u0 = ti * kTile, v0 = tj * kTile;
        double a0[4][4], a1[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) a0[a][b] = a1[a][b] = 0.0;
        int nf = 0;
        for (int f0 = 0; f0 < F; f0 += kF) {
            nf = min(kF, F - f0);
            __syncthreads();
            for (int e = threadIdx.x; e < kTile * kF; e += kThreads) {
                const int r = e / kF, j = e % kF;       // consecutive threads along the features of a frame
                const int64_t u = u0 + r, v = v0 + r;
                sl[j][r] = (j < nf && u < tr.T) ? Xt[u * x_stride + f0 + j] : 0.0;
                sr[j][r] = (j < nf && v < tr.T) ? Xt[v * x_stride + f0 + j] : 0.0;
            }
            __syncthreads();
            for (int j = 0; j + 1 < nf; j += 2) {
                double x0[4], x1[4], y0[4], y1[4];
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    x0[a] = sl[j][ty + 16 * a];
                    x1[a] = sl[j + 1][ty + 16 * a];
                }
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    y0[b] = sr[j][tx + 16 * b];
                    y1[b] = sr[j + 1][tx + 16 * b];
                }
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        a0[a][b] = npy::dadd(a0[a][b], npy::dmul(x0[a], y0[b]));
                        a1[a][b] = npy::dadd(a1[a][b], npy::dmul(x1[a], y1[b]));
                    }
            }
        }
        const bool tail = F & 1;                        // then nf is odd and feature F - 1 sits at nf - 1
        bool any_nan = false;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int64_t u = u0 + ty + 16 * a;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int64_t v = v0 + tx + 16 * b;
                double d = npy::dadd(a0[a][b], a1[a][b]);
                if (tail) d = npy::dadd(d, npy::dmul(sl[nf - 1][ty + 16 * a], sr[nf - 1][tx + 16 * b]));
                if (u >= tr.T || v >= tr.T || u > v) continue;
                if (u == v) {
                    St[u * tr.T + u] = 1.0;
                    continue;
                }
                const double s = similarity(d, nrm[tr.x0 + u], nrm[tr.x0 + v]);
                any_nan |= s != s;
                St[u * tr.T + v] = s;
                St[v * tr.T + u] = s;
            }
        }
        if (any_nan) nan_flag[blockIdx.y] = 1;
    }
}

// Only for a track whose S holds a NaN: Hn[a, j] = 1 when S[a, j .. j + m - 1] holds one (a < T, j < R)
__global__ void __launch_bounds__(256) thumb_nan_window_kernel(const thumb::Track *__restrict__ tracks,
                                                               const double *__restrict__ S, int m,
                                                               const int32_t *__restrict__ nan_flag,
                                                               unsigned char *__restrict__ Hn)
{
    if (!nan_flag[blockIdx.y]) return;
    const thumb::Track tr = tracks[blockIdx.y];
    const double *St = S + tr.s0;
    for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < tr.T * tr.R; e += int64_t(gridDim.x) * blockDim.x) {
        const int64_t a = e / tr.R, j = e - a * tr.R;
        bool nan = false;
        for (int k = 0; k < m; ++k) nan |= St[a * tr.T + j + k] != St[a * tr.T + j + k];
        Hn[tr.h0 + e] = nan;
    }
}

__device__ inline uint64_t warp_min(uint64_t k)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const uint64_t q = __shfl_xor_sync(0xffffffffu, static_cast<unsigned long long>(k), o);
        k = q < k ? q : k;
    }
    return k;
}

// One 32 x 32 tile of a track's C per CTA, upper-triangle tiles only: each entry's diagonal sum (NaN when its box holds
// one), written at (i, j) and (j, i); the tile's min key goes into the track's min by one atomicMin.
__global__ void __launch_bounds__(256) thumb_filter_kernel(const thumb::Track *__restrict__ tracks,
                                                           const double *__restrict__ S, int m,
                                                           const int32_t *__restrict__ nan_flag,
                                                           const unsigned char *__restrict__ Hn, double *__restrict__ C,
                                                           unsigned long long *__restrict__ keys)
{
    using namespace thumb;
    __shared__ uint64_t warp_mins[8];
    const Track tr = tracks[blockIdx.y];
    const bool check_box = nan_flag[blockIdx.y];
    const int64_t nt = (tr.R + kFTile - 1) / kFTile;
    const double *St = S + tr.s0;
    double *Ct = C + tr.c0;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    auto at = [St, &tr](int64_t a, int64_t b) { return St[a * tr.T + b]; };
    uint64_t kmin = ~uint64_t(0);
    for (int64_t l = blockIdx.x; l < upper_tiles(nt); l += gridDim.x) {
        int64_t ti, tj;
        upper_tile(l, nt, ti, tj);
        const int64_t j = tj * kFTile + tx;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int64_t i = ti * kFTile + ty + 8 * a;
            if (i > j || j >= tr.R) continue;
            double c = diag_sum(at, i, j, m);
            if (check_box) {
                bool nan = false;
                for (int k = 0; k < m; ++k) nan |= Hn[tr.h0 + (i + k) * tr.R + j] != 0;
                if (nan) c = double_of(0x7ff8000000000000ull);
            }
            Ct[i * tr.R + j] = c;
            Ct[j * tr.R + i] = c;
            const uint64_t kc = min_key(c);
            kmin = kc < kmin ? kc : kmin;
        }
    }
    kmin = warp_min(kmin);
    if (tx == 0) warp_mins[ty] = kmin;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) kmin = warp_mins[w] < kmin ? warp_mins[w] : kmin;
        atomicMin(keys + blockIdx.y, static_cast<unsigned long long>(kmin));
    }
}

struct Best {
    uint64_t key;
    int64_t idx;
};
__device__ inline Best best_of(Best p, Best q) { return thumb::better(q.key, q.idx, p.key, p.idx) ? q : p; }
__device__ inline Best warp_best(Best p)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        Best q;
        q.key = __shfl_xor_sync(0xffffffffu, static_cast<unsigned long long>(p.key), o);
        q.idx = __shfl_xor_sync(0xffffffffu, static_cast<long long>(p.idx), o);
        p = best_of(p, q);
    }
    return p;
}
// the block's best (threads of 256); every thread gets it
__device__ inline Best block_best(Best p)
{
    __shared__ Best warp_bests[8];
    p = warp_best(p);
    if ((threadIdx.x & 31) == 0) warp_bests[threadIdx.x >> 5] = p;
    __syncthreads();
    p = warp_bests[0];
    for (int w = 1; w < 8; ++w) p = best_of(p, warp_bests[w]);
    return p;
}
// below every key (a NaN-free value's is at least 1)
__device__ inline Best no_best() { return Best{0, INT64_MAX}; }

// The masks applied in place (masked entries become min_sm) and the argmax key over them; each CTA writes its best to
// part[blockIdx.y * gridDim.x + blockIdx.x].
__global__ void __launch_bounds__(thumb::kMaskThreads) thumb_mask_kernel(const thumb::Track *__restrict__ tracks,
                                                                        double gap,
                                                                        const unsigned long long *__restrict__ keys,
                                                                        double *__restrict__ C, Best *__restrict__ part)
{
    using namespace thumb;
    const Track tr = tracks[blockIdx.y];
    const double min_sm = min_value(keys[blockIdx.y]);
    double *Ct = C + tr.c0;
    Best b = no_best();
    for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < tr.R * tr.R; e += int64_t(gridDim.x) * blockDim.x) {
        const int64_t i = e / tr.R, j = e - i * tr.R;
        double v = Ct[e];
        if (masked(i, j, gap, tr.lo, tr.hi)) Ct[e] = v = min_sm;
        b = best_of(b, Best{max_key(v), e});
    }
    b = block_best(b);
    if (threadIdx.x == 0) part[blockIdx.y * int64_t(gridDim.x) + blockIdx.x] = b;
}

// One CTA per track: the argmax from the mask kernel's n_part bests, then the walk (one thread) into idx[4 * track]
__global__ void __launch_bounds__(256) thumb_walk_kernel(const thumb::Track *__restrict__ tracks, int m,
                                                         const Best *__restrict__ part, int n_part,
                                                         const double *__restrict__ C, int64_t *__restrict__ idx)
{
    const thumb::Track tr = tracks[blockIdx.x];
    Best b = no_best();
    for (int p = threadIdx.x; p < n_part; p += blockDim.x) b = best_of(b, part[blockIdx.x * int64_t(n_part) + p]);
    b = block_best(b);
    if (threadIdx.x != 0) return;
    const double *Ct = C + tr.c0;
    thumb::walk([Ct, &tr](int64_t i, int64_t j) { return Ct[i * tr.R + j]; }, tr.R, b.idx / tr.R, b.idx % tr.R, m,
                idx + 4 * int64_t(blockIdx.x));
}

// blocks per track of a grid-striding launch over n_tracks tracks needing at most `need` blocks each
static unsigned blocks_per_track(int64_t need, int64_t n_tracks)
{
    return unsigned(std::max<int64_t>(1, std::min<int64_t>(need, std::max<int64_t>(1, 16384 / n_tracks))));
}

extern "C" int b200aa_music_thumbnail(const double *d_X, int n_feats, int64_t x_stride, const int64_t *h_frames,
                                      int64_t n_tracks, int filter_len, double diag_gap, const int64_t *h_limits,
                                      double *d_sim, double *d_out, int64_t *d_idx, void *stream)
{
    NvtxRange nvtx_("b200aa_music_thumbnail");
    REFUSE_CAPTURE(stream, "b200aa_music_thumbnail", kWhyHostArrays);
    using thumb::Track;
    const int F = n_feats, m = filter_len;
    const bool sim_only = d_sim != nullptr;
    if (!d_X || !h_frames || F < 1 || x_stride < F || n_tracks < 1)
        return B200AA_ERR_INVALID;
    if (sim_only ? (d_out || d_idx) : (!d_out || !d_idx || !h_limits || m < 1))
        return B200AA_ERR_INVALID;
    std::vector<Track> tracks(static_cast<size_t>(n_tracks));
    int64_t rows = 0, c0 = 0;
    for (int64_t b = 0; b < n_tracks; ++b) {
        Track &t = tracks[size_t(b)];
        t.T = h_frames[b];
        if (t.T < 1 || (!sim_only && t.T < m) || t.T > (int64_t(1) << 28)) return B200AA_ERR_INVALID;
        t.x0 = rows;
        t.R = sim_only ? t.T : t.T - m + 1;
        t.lo = sim_only ? 0 : h_limits[2 * b];
        t.hi = sim_only ? t.R : h_limits[2 * b + 1];
        if (t.lo < 0 || t.lo > t.R || t.hi < 0 || t.hi > t.R) return B200AA_ERR_INVALID;
        t.c0 = c0;
        rows += t.T;
        c0 += t.R * t.R;
    }

    // slices of whole tracks whose S and NaN windows fit kScratchSliceBytes; a larger track is a slice of its own
    std::vector<int64_t> cut(1, 0);
    Layout slice_l;
    size_t largest_slice = 0;
    for (int64_t b = 0; b < n_tracks; ++b) {
        Track &t = tracks[size_t(b)];
        const size_t sb = sim_only ? 0 : size_t(t.T * t.T) * sizeof(double), hb = sim_only ? 0 : size_t(t.T * t.R);
        if (b > cut.back() && (slice_l.bytes() + align256(sb) + align256(hb) > kScratchSliceBytes || b - cut.back() == 65535)) {
            cut.push_back(b);
            slice_l = Layout();
        }
        const size_t s_at = slice_l.add(sb);
        t.s0 = sim_only ? t.c0 : int64_t(s_at / sizeof(double));
        t.h0 = int64_t(slice_l.add(hb));
        largest_slice = std::max(largest_slice, slice_l.bytes());
    }
    cut.push_back(n_tracks);
    int64_t max_part = 0;
    for (size_t s = 0; s + 1 < cut.size(); ++s) {
        int64_t maxR = 0;
        for (int64_t b = cut[s]; b < cut[s + 1]; ++b) maxR = std::max(maxR, tracks[size_t(b)].R);
        const int64_t n = cut[s + 1] - cut[s];
        max_part = std::max(max_part, n * blocks_per_track((maxR * maxR + thumb::kMaskThreads - 1) / thumb::kMaskThreads, n));
    }

    // the memsets of the NaN flags and min keys cover their regions' padding too
    Layout L;
    const size_t tracks_at = L.add(tracks.size() * sizeof(Track)), nrm_at = L.add(size_t(rows) * sizeof(double)),
                 flag_at = L.add(size_t(n_tracks) * sizeof(int32_t)), key_at = L.add(size_t(n_tracks) * sizeof(uint64_t)),
                 part_at = L.add(sim_only ? 0 : size_t(max_part) * sizeof(Best)), slice_at = L.add(largest_slice);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(L.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const Track *d_tracks = Layout::at<const Track>(base, tracks_at);
    double *nrm = Layout::at<double>(base, nrm_at);
    int32_t *flag = Layout::at<int32_t>(base, flag_at);
    unsigned long long *keys = Layout::at<unsigned long long>(base, key_at);
    Best *part = Layout::at<Best>(base, part_at);
    char *slice = Layout::at<char>(base, slice_at);
    double *S = sim_only ? d_sim : reinterpret_cast<double *>(slice);
    CK(cudaMemcpyAsync(base, tracks.data(), tracks.size() * sizeof(Track), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(flag, 0, key_at - flag_at, st));
    CK(cudaMemsetAsync(keys, 0xff, part_at - key_at, st));
    thumb_norm_kernel<<<unsigned(std::min<int64_t>((rows + 255) / 256, 1 << 16)), 256, 0, st>>>(d_X, x_stride, F, rows, nrm);
    CK_LAUNCH("thumb_norm_kernel");
    for (size_t s = 0; s + 1 < cut.size(); ++s) {
        const int64_t t0 = cut[s], n = cut[s + 1] - t0;
        int64_t maxT = 0, maxR = 0;
        for (int64_t b = t0; b < t0 + n; ++b) {
            maxT = std::max(maxT, tracks[size_t(b)].T);
            maxR = std::max(maxR, tracks[size_t(b)].R);
        }
        const Track *tr = d_tracks + t0;
        const dim3 g_sim(blocks_per_track(thumb::upper_tiles((maxT + thumb::kTile - 1) / thumb::kTile), n), unsigned(n));
        thumb_sim_kernel<<<g_sim, thumb::kThreads, 0, st>>>(tr, d_X, x_stride, F, nrm, S, flag + t0);
        CK_LAUNCH("thumb_sim_kernel");
        if (sim_only) continue;
        unsigned char *Hn = reinterpret_cast<unsigned char *>(slice);
        const dim3 g_win(blocks_per_track((maxT * maxR + 255) / 256, n), unsigned(n));
        thumb_nan_window_kernel<<<g_win, 256, 0, st>>>(tr, S, m, flag + t0, Hn);
        CK_LAUNCH("thumb_nan_window_kernel");
        const dim3 g_filter(blocks_per_track(thumb::upper_tiles((maxR + thumb::kFTile - 1) / thumb::kFTile), n), unsigned(n));
        thumb_filter_kernel<<<g_filter, 256, 0, st>>>(tr, S, m, flag + t0, Hn, d_out, keys + t0);
        CK_LAUNCH("thumb_filter_kernel");
        const unsigned n_part = blocks_per_track((maxR * maxR + thumb::kMaskThreads - 1) / thumb::kMaskThreads, n);
        thumb_mask_kernel<<<dim3(n_part, unsigned(n)), thumb::kMaskThreads, 0, st>>>(tr, diag_gap, keys + t0, d_out, part);
        CK_LAUNCH("thumb_mask_kernel");
        thumb_walk_kernel<<<unsigned(n), 256, 0, st>>>(tr, m, part, int(n_part), d_out, d_idx + 4 * t0);
        CK_LAUNCH("thumb_walk_kernel");
    }
    return scratch.done(B200AA_OK);
}
