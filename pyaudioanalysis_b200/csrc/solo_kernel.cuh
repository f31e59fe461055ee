// Warp-autonomous short-term kernel for windows N = 2 * L * R2 that are not multiples of 32: 882 = 2 * 21 * 21 (20 ms at
// 44.1 kHz: BASELINE configs[2]), 400 = 2 * 20 * 10, 600 = 2 * 20 * 15.
//
// Same organisation as the pair kernel (csrc/pair_kernel.cuh): one warp owns a run of consecutive frames, two frames
// (2q, 2q + 1) per step, no CTA-wide barrier, the feature phases are the pair kernel's (rows_to_features, tile_store).
// The transform differs: every frame gets its OWN packed-real FFT of Nc = L * R2 complex points
// z[m] = (x[2m] - x[0]) + i (x[2m+1] - x[0]);  m = L n1 + n2, k = k1 + R2 k2:  lane n2 < L runs the R2-point transform over
// n1 in registers, twiddles by W_Nc^(n2 k1), one transpose through shared memory, lane k1 < R2 runs the L-point transform
// over n2, Z lands in natural order and each lane turns (Z[k], Z[Nc-k]) pairs into |X[k]| and |X[Nc-k]| with one twiddle
// W_N^k.  Time-domain rows use the pair kernel's row layout (lane = sample mod 32, whole frames, last row partial).
// MODE = spectrogram / chromagram writes rows [R x K] / [R x 12] instead of features (no halo, no time-domain work).
#pragma once
#include "pair_kernel.cuh"

namespace b200aa {

template <int L, int R2>
struct SoloShape {
    static constexpr int Nc = L * R2, N = 2 * Nc, K = Nc, Kp = DenseShape<K>::Kp, C = Kp / 32;
    static constexpr int RT = (N + 31) / 32;             // 32-sample rows of a frame; the last one holds LASTV samples
    static constexpr int LASTV = N - 32 * (RT - 1);
    static constexpr int TS = L | 1;                     // row stride (float2) of the transposed pass-1 outputs: odd
    static constexpr int TZ = (R2 * TS > Nc + 2) ? R2 * TS : Nc + 2;
    static constexpr int Lt = N / 10;
    static constexpr int NREST = (N % 10) ? 1 : 0, NE = 10 + NREST;
    static constexpr int KH = (Nc - 1) / 2;              // pairs (k, Nc - k), k = 1 .. KH; Nc even: bin Nc / 2 pairs with itself
    // feature layout: after frame b's transform its |X| row, the mel scratch, the entropy parts and the chroma sums live in the
    // transform buffer (floats): a warp keeps only frame a's row, the previous b row, the feature tile and the block energies beside it
    static constexpr int MS0 = (Kp + 3) & ~3;
    static constexpr int PT0 = MS0 + 6 * B200AA_N_MEL, CH0 = PT0 + 64;
    static constexpr int TZF = (2 * TZ >= CH0 + 24) ? TZ : (CH0 + 24 + 1) / 2;      // float2 elements of the feature layout's buffer
    static_assert(L <= 32 && R2 <= 32, "one lane per column / row");
    static_assert(Lt >= 32 && (Lt % 2) == 0, "a 32-sample row touches two energy blocks at most");
};

template <int L, int R2>
struct alignas(16) SoloWarpMem {
    using S = SoloShape<L, R2>;
    float2 tz[S::TZF];                       // pass-1 outputs [k1][TS]  ->  Z[k] (natural order)  ->  (after frame b) |X| row of b | mel scratch | parts | chroma
    alignas(16) float rowa[S::Kp];           // |X| row of frame a
    alignas(16) float rowp[S::Kp];           // |X| row of the previous step's frame b
    float fv[9 * kFvStride];
    float blk[24];                           // block energies: a -> [0, 10), b -> [10, 20), rests at 20, 21
};

// the row modes (spectrogram / chromagram) keep only the transform buffer and the two |X| rows: small CTAs, more of them per SM
// (the spectrogram stores its rows straight to global memory and keeps the transform buffer only)
template <int L, int R2, int MODE>
struct alignas(16) SoloRowWarpMem {
    using S = SoloShape<L, R2>;
    float2 tz[S::TZ];
    alignas(16) float rows[2][MODE == kModeChromagram ? S::Kp : 4];
};
template <int L, int R2, int MODE> struct SoloWarpMemFor { using type = SoloRowWarpMem<L, R2, MODE>; };
template <int L, int R2> struct SoloWarpMemFor<L, R2, kModeFeatures> { using type = SoloWarpMem<L, R2>; };

// the feature layout: one CTA of 24 warps at 80 registers; config 3 (64 x 60 s @44.1 kHz, 882 / 441) on an H100 80GB HBM3
// (700 W): 1 x 24 1.297 ms, 1 x 16 1.281 ms (within the spread of one run)
#ifndef B200AA_SOLO_MAXWARPS
#define B200AA_SOLO_MAXWARPS 24
#endif
#ifndef B200AA_SOLO_MINBLOCKS
#define B200AA_SOLO_MINBLOCKS 1
#endif
constexpr int kSoloMaxWarps = B200AA_SOLO_MAXWARPS, kSoloMinBlocks = B200AA_SOLO_MINBLOCKS;
// Measured on config 3 (64 x 60 s @44.1 kHz), warps per CTA x CTAs per SM -> spectrogram / chromagram ms:
//   8 x 2 (126 regs, the feature layout) 0.558 / 0.592    5 x 4 (96 regs) 0.543 / 0.558    8 x 3 (80 regs) 0.502 / 0.537
//   6 x 4 (80) 0.499 / 0.546    7 x 4 (71) 0.490 / 0.561    10 x 3 (64) 0.485 / 0.565    8 x 4 (64 regs, 32 warps) 0.478 / 0.552
// (the chromagram's two |X| rows per warp cap it at 3 CTAs of 8 warps)
#ifndef B200AA_SOLO_ROW_WARPS
#define B200AA_SOLO_ROW_WARPS 8
#endif
#ifndef B200AA_SOLO_SPEC_BLOCKS
#define B200AA_SOLO_SPEC_BLOCKS 4
#endif
#ifndef B200AA_SOLO_CHROMA_BLOCKS
#define B200AA_SOLO_CHROMA_BLOCKS 3
#endif
constexpr int kSoloRowWarps = B200AA_SOLO_ROW_WARPS;
constexpr int kSoloCtaCap = (kSoloMinBlocks == 1 ? 227 : (kSoloMinBlocks == 2 ? 113 : 228 / kSoloMinBlocks - 1)) * 1024;   // feature layout

template <int L, int R2, int MODE = kModeFeatures>
__host__ __device__ constexpr int solo_warps()
{
    if (MODE != kModeFeatures) return kSoloRowWarps;
    constexpr int budget = kSoloCtaCap - (L * R2 + L * R2 / 2 + 2) * 8 - 256 - 6656;
    constexpr int w = budget / int(sizeof(SoloWarpMem<L, R2>));
    constexpr int c = w > kSoloMaxWarps ? kSoloMaxWarps : (w < 2 ? 2 : w);
    return c >= 4 ? (c & ~3) : c;            // whole rounds over the four schedulers
}
template <int MODE>
__host__ __device__ constexpr int solo_min_blocks()
{
    return MODE == kModeFeatures ? kSoloMinBlocks : (MODE == kModeSpectrogram ? B200AA_SOLO_SPEC_BLOCKS : B200AA_SOLO_CHROMA_BLOCKS);
}

template <int L, int R2, int MODE = kModeFeatures>
struct alignas(16) SoloCtaMem {
    using S = SoloShape<L, R2>;
    float2 tw[R2 * L];                       // W_Nc^(k1 n2), [k1][n2]
    float2 twp[(S::Nc / 2 + 2) & ~1];        // W_N^k, k <= Nc / 2
    alignas(16) int dlane[16 * 4];
    typename SoloWarpMemFor<L, R2, MODE>::type w[solo_warps<L, R2, MODE>()];
};

struct SoloParams {
    StParams st;
    const float2 *tw, *twp;
    const int *pblob;
    PairBlobLayout pbl;
    unsigned int *counter;                              // row modes: work counter over the run list below
    int seg_big, n_big, seg_small, segs_per_clip;       // row modes: runs of pairs per clip, long ones first (rows need no halo)
    StealParams sched;                                  // features: static shares + steal-half (sched.cuh), as in the pair kernel
};

template <int L, int R2, int MODE = kModeFeatures>
inline size_t solo_smem_bytes(int blob_words)
{
    return sizeof(SoloCtaMem<L, R2, MODE>) + (MODE == kModeSpectrogram ? 0 : sizeof(int) * size_t((blob_words + 3) & ~3));   // no tables
}

// time-domain accumulation of BOTH frames over all rows (u[r] = (sample of a, sample of b) of lane l = sample 32 r + l);
// see td_pair in pair_kernel.cuh -- this form takes any window length (the last row is partial)
template <int L, int R2, bool TWO>
__device__ __forceinline__ void td_rows(const float2 (&u)[SoloShape<L, R2>::RT], float cm, const b200aa_clip_norm &nm, int lane,
                                        float2 *e2, int &flips_a, int &flips_b)
{
    using S = SoloShape<L, R2>;
    constexpr int N = S::N, Lt = S::Lt, RT = S::RT;
    unsigned pPa = 0u, pQa = 0u, pPb = 0u, pQb = 0u;
    int fa = 0, fb = 0;
    const float2 ncm = make_float2(-cm, -cm), a2 = make_float2(nm.a, nm.a), bp2 = make_float2(nm.bp, nm.bp);
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        const bool live = r < RT - 1 || lane < S::LASTV;
        const float2 d = f2add(u[r], ncm);
        const unsigned Pa = __ballot_sync(0xffffffffu, live && d.x > nm.lo), Pb = __ballot_sync(0xffffffffu, live && d.y > nm.lo);
        unsigned Qa = 0u, Qb = 0u;
        if (TWO) { Qa = __ballot_sync(0xffffffffu, live && d.x < nm.hi); Qb = __ballot_sync(0xffffffffu, live && d.y < nm.hi); }
        if (r == 0) { pPa = (Pa & 1u) << 31; pQa = (Qa & 1u) << 31; pPb = (Pb & 1u) << 31; pQb = (Qb & 1u) << 31; }
        const unsigned valid = (r == RT - 1 && S::LASTV < 32) ? ((1u << S::LASTV) - 1u) : 0xffffffffu;
        fa += __popc((Pa ^ __funnelshift_l(pPa, Pa, 1)) & valid);
        fb += __popc((Pb ^ __funnelshift_l(pPb, Pb, 1)) & valid);
        if (TWO) {
            fa += __popc((Qa ^ __funnelshift_l(pQa, Qa, 1)) & valid);
            fb += __popc((Qb ^ __funnelshift_l(pQb, Qb, 1)) & valid);
        }
        const float2 y = f2fma(a2, d, bp2);
        const int n0 = 32 * r;
        const int b0 = (n0 / Lt) < 10 ? (n0 / Lt) : 10;
        const int end = b0 < 10 ? (b0 + 1) * Lt : N;
        const int thr = end - n0;
        const int i0 = b0, i1 = (b0 + 1 < 10 ? b0 + 1 : 10);
        if (thr >= 32) {
            if (i0 < S::NE) { if (live) e2[i0] = f2fma(y, y, e2[i0]); }
        } else {
            const bool first = lane < thr;
            if (i0 < S::NE) { if (live && first) e2[i0] = f2fma(y, y, e2[i0]); }
            if (i1 < S::NE) { if (live && !first) e2[i1] = f2fma(y, y, e2[i1]); }
        }
        pPa = Pa; pQa = Qa; pPb = Pb; pQb = Qb;
    }
    flips_a = TWO ? fa : 2 * fa;
    flips_b = TWO ? fb : 2 * fb;
}

// RAGGED (row modes only): every clip takes its own row counts from p.len (ragged_rows); a template flag so that the
// uniform launches keep their code.
template <int L, int R2, int MODE, bool RAGGED = false>
__global__ void __launch_bounds__(32 * solo_warps<L, R2, MODE>(), solo_min_blocks<MODE>()) st_solo_kernel(const SoloParams pp)
{
    using S = SoloShape<L, R2>;
    constexpr int Nc = S::Nc, N = S::N, K = S::K, Kp = S::Kp, RT = S::RT, TS = S::TS, KH = S::KH;
    constexpr int NTHR = 32 * solo_warps<L, R2, MODE>();
    constexpr bool FEAT = MODE == kModeFeatures;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SoloCtaMem<L, R2, MODE> &cm_ = *reinterpret_cast<SoloCtaMem<L, R2, MODE> *>(smem_raw);
    int *const blob_s = reinterpret_cast<int *>(smem_raw + sizeof(SoloCtaMem<L, R2, MODE>));
    const StParams &p = pp.st;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if constexpr (MODE != kModeSpectrogram) { for (int i = tid; i < pp.pbl.words; i += NTHR) blob_s[i] = pp.pblob[i]; }
    for (int i = tid; i < R2 * L; i += NTHR) cm_.tw[i] = pp.tw[i];
    for (int i = tid; i < Nc / 2 + 1; i += NTHR) cm_.twp[i] = pp.twp[i];
    if (tid < 16) *reinterpret_cast<int4 *>(cm_.dlane + tid * 4) = pair_lane_init<K>(tid);
    __syncthreads();
    const FeatTables ftab{reinterpret_cast<const float *>(blob_s + pp.pbl.dct), blob_s + pp.pbl.mel_rec,
                          reinterpret_cast<const float4 *>(blob_s + pp.pbl.mel_w), reinterpret_cast<const int2 *>(blob_s + pp.pbl.chr),
                          pp.pbl.lq, pp.pbl.ct};
    auto &wm = cm_.w[warp];
    const int step = p.step;
    const int half = lane >> 4, l16 = lane & 15;
    const unsigned FULLM = 0xffffffffu;

    // ---- features: the run in progress (warp-uniform; see pair_kernel.cuh)
    unsigned g0 = 0, g1 = 0, inc = FEAT ? pp.sched.chunk : 0u;
    unsigned run_b = 0xffffffffu, run_q = 0xffffffffu;
    int tile_n = 0, tile_t0 = 0;
    if constexpr (FEAT) {
        if (lane == 0) sched_begin(pp.sched, blockIdx.x * unsigned(solo_warps<L, R2, MODE>()) + unsigned(warp));
        __syncwarp();
    }
#define B200AA_SOLO_FLUSH(clip_index) tile_flush(wm.fv, tile_n, tile_t0, p.out + size_t(clip_index) * p.n_out * p.t_stride, p.t_stride, p.n_out, lane)

    for (;;) {
        int64_t b;
        int q0, q1, T, NP;
        int64_t valid_b = 0;        // row modes: rows of clip b from full frames
        bool fresh = true;
        if constexpr (FEAT) {
            if (g0 >= g1) {
                const int got = sched_next(pp.sched, blockIdx.x * unsigned(solo_warps<L, R2, MODE>()) + unsigned(warp), lane, inc, g0, g1);
                if (got == 0) break;
                if (got == 2) continue;
            }
            const unsigned per_clip = pp.sched.per_clip;
            const unsigned cb = g0 / per_clip;
            q0 = int(g0 - cb * per_clip);
            int qe = q0 + int(g1 - g0);
            qe = qe < int(per_clip) ? qe : int(per_clip);
            g0 += unsigned(qe - q0);                                // a chunk may run over the end of a clip
            b = int64_t(cb);
            const bool cont = cb == run_b && unsigned(q0) == run_q; // the run goes on: state carried, no halo
            if (!cont) { B200AA_SOLO_FLUSH(run_b); tile_t0 = 2 * q0; }
            fresh = !cont;
            run_b = cb;
            run_q = 0xffffffffu;
            const int64_t len = p.len ? p.len[b] : p.n_samples;
            T = int(len < N ? 0 : (len - N) / step + 1);
            NP = (T + 1) >> 1;
            if (q0 >= NP) continue;                                 // ragged batch: beyond this clip's last pair
            q1 = qe < NP ? qe : NP;
        } else {
            unsigned item = 0;
            if (lane == 0) item = atomicAdd(pp.counter, 1u);
            item = __shfl_sync(FULLM, item, 0);
            if (int64_t(item) >= p.n_items) break;
            const int seg = int(item / unsigned(p.n_clips));
            b = item - unsigned(seg) * unsigned(p.n_clips);
            int64_t rows_b = p.rows_launch;                         // the rows of this launch (rows >= rows_valid are zero)
            valid_b = p.rows_valid;
            if constexpr (RAGGED) ragged_rows<MODE>(p, b, rows_b, valid_b);
            T = int(rows_b);
            NP = (T + 1) >> 1;
            if (seg < pp.n_big) { q0 = seg * pp.seg_big; q1 = q0 + pp.seg_big; }
            else { q0 = pp.n_big * pp.seg_big + (seg - pp.n_big) * pp.seg_small; q1 = q0 + pp.seg_small; }
            if (q0 >= NP) continue;
            q1 = q1 < NP ? q1 : NP;
        }
        const int n_valid = MODE == kModeFeatures ? T : int(valid_b);
        const b200aa_clip_norm nm = p.norm[b];
        const bool is16 = p.dtype == B200AA_DTYPE_I16;
        const char *clip = reinterpret_cast<const char *>(p.sig) + size_t(b) * p.clip_stride * (is16 ? 2 : 4);
        const float M0 = is16 ? 8421376.f : 0.f;                   // u = M0 + x exactly (2^23 + 2^15 trick for int16)
        const float cmv = M0 + nm.m;
        const bool two_sided = !(nm.hi > nm.lo);
        const float sc = nm.a / float(2 * K);
        const unsigned short *const c16 = reinterpret_cast<const unsigned short *>(clip);
        const float *const c32 = reinterpret_cast<const float *>(clip);
        // sample n of the clip as the exact float M0 + x
        auto s16 = [&](int64_t n) -> float { return __int_as_float(0x4B000000 | (int(__ldg(c16 + n)) ^ 0x8000)); };
        auto s32 = [&](int64_t n) -> float { return __ldg(c32 + n); };

        const int halo = (MODE == kModeFeatures && fresh && q0 > 0) ? 1 : 0;
        for (int q = q0 - halo; q < q1; ++q) {
            const bool store = q >= q0;
            const int ta = 2 * q;
            const bool bvalid = ta + 1 < T;
            const int tbb = bvalid ? ta + 1 : ta;
            const int64_t sa0 = frame_first<MODE>(N, step, ta), sb0 = frame_first<MODE>(N, step, tbb);       // first samples
            float *rowa, *rowb;              // features: frame b's row lands in the transform buffer once its transform is done
            if constexpr (FEAT) { rowa = wm.rowa; rowb = reinterpret_cast<float *>(wm.tz); }
            else { rowa = wm.rows[0]; rowb = wm.rows[1]; }
            const int ra = store ? 1 + tile_n : 8, rb = store ? 2 + tile_n : 0;
            const bool a_real = MODE == kModeFeatures || ta < n_valid, b_real = MODE == kModeFeatures || tbb < n_valid;

            // ---- time-domain rows (features only): whole frames in the row layout
            if constexpr (MODE == kModeFeatures) {
                float2 u[RT];
                if (is16) {
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        const bool live = r < RT - 1 || lane < S::LASTV;
                        u[r] = live ? make_float2(s16(sa0 + 32 * r + lane), s16(sb0 + 32 * r + lane)) : make_float2(cmv, cmv);
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        const bool live = r < RT - 1 || lane < S::LASTV;
                        u[r] = live ? make_float2(s32(sa0 + 32 * r + lane), s32(sb0 + 32 * r + lane)) : make_float2(cmv, cmv);
                    }
                }
                float2 e2[S::NE];
#pragma unroll
                for (int i = 0; i < S::NE; ++i) e2[i] = make_float2(0.f, 0.f);
                int fl_a, fl_b;
                if (two_sided) td_rows<L, R2, true>(u, cmv, nm, lane, e2, fl_a, fl_b);
                else td_rows<L, R2, false>(u, cmv, nm, lane, e2, fl_a, fl_b);
                float ev[2 * S::NE];
#pragma unroll
                for (int i = 0; i < S::NE; ++i) { ev[i] = e2[i].x; ev[S::NE + i] = e2[i].y; }
                MultiReduce<2 * S::NE>::run(ev, lane);
                __syncwarp();
                {
                    constexpr int SH = MultiReduce<2 * S::NE>::SH;
                    const int j = lane >> SH;
                    if ((lane & ((1 << SH) - 1)) == 0 && j < 2 * S::NE) {
                        const int f = j >= S::NE ? 1 : 0, i = j - f * S::NE;
                        wm.blk[i < 10 ? 10 * f + i : 20 + f] = ev[0];
                    }
                }
                __syncwarp();
                const bool own = l16 < 10;
                const float e = own ? wm.blk[half * 10 + l16] : 0.f;
                float tot = half_sum(e);
                if (S::NREST) tot += wm.blk[20 + half];
                const float sj = fdiv(e, tot + B200AA_EPS);
                const float H = half_sum(own ? -sj * flog2(sj + B200AA_EPS) : 0.f);
                if (l16 == 0) {
                    float *fv = wm.fv + (half ? rb : ra) * kFvStride;
                    fv[0] = float(half ? fl_b : fl_a) * 0.5f / float(N - 1);
                    fv[1] = tot / float(N);
                    fv[2] = H;
                }
            }

            // ---- one packed-real transform per frame
            // samples of a frame in transform layout: lane n2 < L holds z[L n1 + n2] = (x[2m] - x0) + i (x[2m+1] - x0), n1 < R2
            auto load_points = [&](int64_t s0, float u0, float2 (&z)[R2]) {
                const int n2 = lane < L ? lane : 0;
                const float2 nu0 = make_float2(-u0, -u0);
                if (is16) {
#pragma unroll
                    for (int n1 = 0; n1 < R2; ++n1) {
                        const int64_t m = s0 + 2 * (L * n1 + n2);
                        z[n1] = f2add(make_float2(s16(m), s16(m + 1)), nu0);
                    }
                } else {
#pragma unroll
                    for (int n1 = 0; n1 < R2; ++n1) {
                        const int64_t m = s0 + 2 * (L * n1 + n2);
                        z[n1] = f2add(make_float2(s32(m), s32(m + 1)), nu0);
                    }
                }
            };
            // both passes + post-processing; the |X| row goes to shared memory, or (gdst != nullptr) straight to global memory
            auto transform = [&](float2 (&z)[R2], float u0, float *row, float *gdst) {
                fft_r<R2>(z);
                if (lane < L) {
                    wm.tz[lane] = z[0];
#pragma unroll
                    for (int k1 = 1; k1 < R2; ++k1) wm.tz[k1 * TS + lane] = cmul(z[k1], cm_.tw[k1 * L + lane]);
                }
                __syncwarp();
                {   // pass 2: lane k1 < R2, L points over n2 -> Z[k1 + R2 k2]
                    float2 v[L];
                    const int k1 = lane < R2 ? lane : 0;
#pragma unroll
                    for (int n2 = 0; n2 < L; ++n2) v[n2] = wm.tz[k1 * TS + n2];
                    fft_r<L>(v);
                    __syncwarp();
                    if (lane < R2) {
#pragma unroll
                        for (int k2 = 0; k2 < L; ++k2) wm.tz[lane + R2 * k2] = v[k2];
                    }
                }
                __syncwarp();
                // post-processing: (Z[k], Z[Nc-k]) -> |X[k]|, |X[Nc-k]|  (X = ev + W_N^k od, X' = conj(ev - W_N^k od))
                float *const dst = MODE == kModeSpectrogram ? gdst : row;
                constexpr int NJ = (KH + 31) / 32;
                float vlo[NJ], vhi[NJ];
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    const int k = 1 + lane + 32 * j;
                    vlo[j] = 0.f; vhi[j] = 0.f;
                    if (k <= KH) {
                        const float2 zk = wm.tz[k], zp = wm.tz[Nc - k];
                        const float2 ev = make_float2(zk.x + zp.x, zk.y - zp.y);
                        const float2 od = make_float2(zk.y + zp.y, zp.x - zk.x);
                        const float2 t = cmul(od, cm_.twp[k]);
                        const float ar = ev.x + t.x, ai = ev.y + t.y, br = ev.x - t.x, bi = ev.y - t.y;
                        vlo[j] = fsqrt_fast(fmaf(ar, ar, ai * ai)) * sc;
                        vhi[j] = fsqrt_fast(fmaf(br, br, bi * bi)) * sc;
                        if constexpr (!FEAT) { dst[k] = vlo[j]; dst[Nc - k] = vhi[j]; }
                    }
                }
                float dc = 0.f, mid = 0.f;
                if (lane == 0) {
                    const float2 z0 = wm.tz[0];
                    // DC: a sum(x - x0) + N (a (x0 - m) + bp), over K
                    dc = fabsf(fmaf(nm.a, z0.x + z0.y, float(N) * fmaf(nm.a, u0 - cmv, nm.bp))) / float(K);
                    if ((Nc & 1) == 0) {
                        const float2 zm = wm.tz[Nc / 2];
                        mid = fsqrt_fast(fmaf(zm.x, zm.x, zm.y * zm.y)) * (2.f * sc);
                    }
                }
                if constexpr (FEAT) {
                    // the row may be the transform buffer itself (frame b): every lane has read Z before anybody writes
                    __syncwarp();
#pragma unroll
                    for (int j = 0; j < NJ; ++j) {
                        const int k = 1 + lane + 32 * j;
                        if (k <= KH) { dst[k] = vlo[j]; dst[Nc - k] = vhi[j]; }
                    }
                }
                if (lane == 0) {
                    dst[0] = dc;
                    if ((Nc & 1) == 0) dst[Nc / 2] = mid;
                }
                if constexpr (MODE != kModeSpectrogram) {
                    if (lane < Kp - K) row[K + lane] = 0.f;
                    if (Kp - K > 32 && lane + 32 < Kp - K) row[K + 32 + lane] = 0.f;
                }
                __syncwarp();
            };
            if constexpr (MODE == kModeFeatures) {
#pragma unroll 1
                for (int f = 0; f < 2; ++f) {
                    const int64_t s0 = f ? sb0 : sa0;
                    const float u0 = is16 ? s16(s0) : s32(s0);
                    float2 z[R2];
                    load_points(s0, u0, z);
                    transform(z, u0, f ? rowb : rowa, nullptr);
                }
            } else {
                // row modes: rows the reference's loop never reaches are zeros and touch no sample.  (Measured and rejected:
                // fetching the samples of both frames before the first transform: slower for config 3's spectrogram.)
                float *const g0 = MODE == kModeSpectrogram ? p.out + (size_t(b) * p.rows_launch + ta) * K : nullptr;
#pragma unroll 1
                for (int f = 0; f < 2; ++f) {
                    if (f && !bvalid) break;
                    float *const gd = g0 ? g0 + f * K : nullptr;
                    float *const row = f ? rowb : rowa;
                    if (!(f ? b_real : a_real)) {
                        if constexpr (MODE == kModeSpectrogram) { for (int k = lane; k < K; k += 32) gd[k] = 0.f; }
                        else { for (int k = lane; k < Kp; k += 32) row[k] = 0.f; }
                        continue;
                    }
                    const int64_t s0 = f ? sb0 : sa0;
                    const float u0 = is16 ? s16(s0) : s32(s0);
                    float2 z[R2];
                    load_points(s0, u0, z);
                    transform(z, u0, row, gd);
                }
                __syncwarp();
            }

            if constexpr (MODE == kModeSpectrogram) {
                // rows went straight to global memory
            } else if constexpr (MODE == kModeChromagram) {
                const float *X = half ? rowb : rowa;
                float sxx = 0.f;
#pragma unroll
                for (int i = 0; i < Kp / 16; ++i) { const float v = X[l16 * (Kp / 16) + i]; sxx = fmaf(v, v, sxx); }
                sxx = half_sum(sxx);
                float ch = 0.f;
                for (int t = 0; t < ftab.CT; ++t) {
                    const int2 e = ftab.chr[t * 16 + l16];
                    const float v = X[e.x];
                    ch = fmaf(v * v, __int_as_float(e.y), ch);
                }
                ch = ch / (sxx == 0.f ? B200AA_EPS : sxx);
                if (l16 < 12 && (half == 0 || bvalid))
                    p.out[(size_t(b) * p.rows_launch + ta + half) * 12 + l16] = (half ? b_real : a_real) ? ch : 0.f;
                __syncwarp();
            } else {
                float *const msraw = rowb + S::MS0, *const mslog = msraw + 2 * B200AA_N_MEL, *const mfold = mslog + 2 * B200AA_N_MEL;
                rows_to_features<K>(rowa, rowb, fresh ? rowa : wm.rowp, fresh, wm.fv[(ra - 1) * kFvStride + 34], cm_.dlane,
                                    rowb + S::PT0, msraw, mslog, mfold, rowb + S::CH0, wm.fv + ra * kFvStride, wm.fv + rb * kFvStride, ftab, lane);
                // frame b's row outlives the next transforms beside the buffer (rows_to_features ends with a __syncwarp)
#pragma unroll
                for (int j = 0; j < (Kp / 4 + 31) / 32; ++j) {      // 16 bytes per lane and instruction
                    const int i4 = lane + 32 * j;
                    if (i4 < Kp / 4) reinterpret_cast<float4 *>(wm.rowp)[i4] = reinterpret_cast<const float4 *>(rowb)[i4];
                }
                if (store) {
                    tile_n += bvalid ? 2 : 1;
                    if (tile_n == 8) B200AA_SOLO_FLUSH(b);          // full tiles leave at once, a partial one when the run ends
                }
            }
            fresh = false;
            if constexpr (FEAT) __syncwarp();       // the copy has read the buffer before the next transform overwrites it
        }
        if constexpr (FEAT) {
            if (q1 < NP) run_q = unsigned(q1);
            else B200AA_SOLO_FLUSH(b);              // end of the clip (an odd frame count leaves a partial tile)
        }
    }
    if constexpr (FEAT) B200AA_SOLO_FLUSH(run_b);
#undef B200AA_SOLO_FLUSH
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
inline bool solo_shape_for_window(int window, int *l, int *r2)
{
    switch (window) {
    case 882: *l = 21; *r2 = 21; return true;     // 20 ms @ 44.1 kHz
    case 400: *l = 20; *r2 = 10; return true;     // 25 ms @ 16 kHz, 50 ms @ 8 kHz
    case 600: *l = 20; *r2 = 15; return true;     // 75 ms @ 8 kHz
    default: return false;
    }
}

struct SoloTables {
    b200aa_host::DeviceMemory tw, twp;  // float2 [R2][L], [Nc/2+1]
    b200aa_host::DeviceMemory pblob;    // int [pbl.words]
    PairBlobLayout pbl{};
    int L = 0, R2 = 0;
};

inline int solo_plan_init(int window, const std::vector<int> &h_pblob, const PairBlobLayout &pbl, SoloTables *stb)
{
    int L = 0, R2 = 0;
    stb->L = 0;
    if (!solo_shape_for_window(window, &L, &R2)) return B200AA_OK;
    const int Nc = L * R2, N = 2 * Nc;
    if (b200aa_host::upload(b200aa_host::twiddle_grid(R2, L, Nc), stb->tw) != cudaSuccess ||
        b200aa_host::upload(b200aa_host::twiddles(Nc / 2 + 1, N), stb->twp) != cudaSuccess ||
        b200aa_host::upload(h_pblob, stb->pblob) != cudaSuccess)
        return B200AA_ERR_CUDA;
    stb->pbl = pbl;
    stb->L = L; stb->R2 = R2;
    return B200AA_OK;
}

#ifndef B200AA_LAYOUT_ONLY
template <int L, int R2, int MODE>
inline int solo_launch_t(const SoloTables &stb, const StParams &p, int sm_count, int64_t T, unsigned int *counter, size_t counter_cap,
                         cudaStream_t st)
{
    const size_t smem = solo_smem_bytes<L, R2, MODE>(stb.pbl.words);
    constexpr int cap = MODE == kModeFeatures ? kSoloCtaCap : 113 * 1024;
    if (smem > size_t(cap)) return B200AA_ERR_UNSUPPORTED;
    auto kern = st_solo_kernel<L, R2, MODE>;
    if constexpr (MODE != kModeFeatures) {
        if (p.len) kern = st_solo_kernel<L, R2, MODE, true>;
    }
    constexpr int W = solo_warps<L, R2, MODE>();
    int occ = 1;
    if (resident_ctas(kern, 32 * W, smem, cap, occ) != cudaSuccess) return B200AA_ERR_CUDA;
    SoloParams pp;
    pp.st = p;
    pp.tw = static_cast<const float2 *>(stb.tw.get()); pp.twp = static_cast<const float2 *>(stb.twp.get());
    pp.pblob = static_cast<const int *>(stb.pblob.get()); pp.pbl = stb.pbl;
    pp.counter = counter;
    const int64_t NP = (T + 1) / 2;
    const int64_t slots = int64_t(sm_count) * occ * W;
    const int64_t total = NP * p.n_clips;
    int64_t grid = int64_t(sm_count) * occ;
    if (MODE == kModeFeatures) {
        // static shares + steal-half (sched.cuh): the slot is the per-warp range table
        if (total <= 0) return B200AA_OK;
        const int rc = steal_setup(pp.sched, reinterpret_cast<unsigned long long *>(counter), counter_cap, total, NP, W, grid, st);
        if (rc != B200AA_OK) return rc;
        pp.seg_big = pp.n_big = pp.seg_small = pp.segs_per_clip = 0;
        pp.st.n_items = total;
        if (getenv("B200AA_DEBUG"))
            fprintf(stderr, "[b200aa] solo kernel %dx%d features: smem %zu B, %d CTAs/SM x %d warps, grid %lld, %lld pairs\n", L, R2, smem, occ, W,
                    (long long)grid, (long long)total);
        kern<<<(unsigned)grid, 32 * W, smem, st>>>(pp);
        return cudaPeekAtLastError() == cudaSuccess ? B200AA_OK : B200AA_ERR_CUDA;
    }
    pp.sched = StealParams{};
    int64_t share = (total + slots - 1) / slots;
    if (share < 1) share = 1;
    int64_t small = share / 10;
    small = small < 4 ? 4 : (small > 48 ? 48 : small);
    int64_t big = share / 3;
    big = big < small ? small : big;
    if (big > NP) big = NP;
    if (small > NP) small = NP;
    int64_t n_big = (NP * 3 / 4) / big;
    if (total <= slots * 2) n_big = 0;
    const int64_t left = NP - n_big * big;
    const int64_t n_small = (left + small - 1) / small;
    pp.seg_big = int(big); pp.n_big = int(n_big); pp.seg_small = int(small);
    pp.segs_per_clip = int(n_big + n_small);
    pp.st.n_items = int64_t(pp.segs_per_clip) * p.n_clips;
    if (pp.st.n_items >= (int64_t(1) << 31) || T >= (int64_t(1) << 30)) return B200AA_ERR_UNSUPPORTED;
    grid = (pp.st.n_items + W - 1) / W;
    if (grid > int64_t(sm_count) * occ) grid = int64_t(sm_count) * occ;
    if (grid < 1) grid = 1;
    if (getenv("B200AA_DEBUG"))
        fprintf(stderr, "[b200aa] solo kernel %dx%d mode %d: smem %zu B, %d CTAs/SM x %d warps, grid %lld, %lld items\n", L, R2, MODE, smem, occ, W,
                (long long)grid, (long long)pp.st.n_items);
    if (cudaMemsetAsync(counter, 0, sizeof(unsigned int), st) != cudaSuccess) return B200AA_ERR_CUDA;
    kern<<<(unsigned)grid, 32 * W, smem, st>>>(pp);
    return cudaPeekAtLastError() == cudaSuccess ? B200AA_OK : B200AA_ERR_CUDA;
}

template <int MODE>
inline int solo_launch_mode(const SoloTables &stb, const StParams &p, int sm_count, int64_t T, unsigned int *counter, size_t counter_cap,
                            cudaStream_t st)
{
    if (stb.L == 21 && stb.R2 == 21) return solo_launch_t<21, 21, MODE>(stb, p, sm_count, T, counter, counter_cap, st);
    if (stb.L == 20 && stb.R2 == 10) return solo_launch_t<20, 10, MODE>(stb, p, sm_count, T, counter, counter_cap, st);
    if (stb.L == 20 && stb.R2 == 15) return solo_launch_t<20, 15, MODE>(stb, p, sm_count, T, counter, counter_cap, st);
    return B200AA_ERR_UNSUPPORTED;
}
#endif  // B200AA_LAYOUT_ONLY

}  // namespace b200aa
