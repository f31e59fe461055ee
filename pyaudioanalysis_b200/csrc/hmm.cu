// libb200aa.so -- HMM segmentation (kernel 7).
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/b200aa.h"
#include "entry.h"
#include "hmm.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 7: HMM segmentation (audioSegmentation.py:287-344, :471-492), bit for bit the NumPy restatement (csrc/hmm.cuh)
// ------------------------------------------------------------------------------------------------
// One thread per (class, feature): the class's windows in the concatenated order, a sequential chain (pairwise for F == 1).
// col[i] is the element offset of window i's feature 0; out is [4, C, F]: sum, mean, ssq, std.
template <class T>
__global__ void __launch_bounds__(128) hmm_stats_kernel(const T *__restrict__ mid, int F, int64_t m_stride,
                                                        const int64_t *__restrict__ col, const int64_t *__restrict__ class_off,
                                                        int C, double *__restrict__ out)
{
    const int64_t w = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (w >= int64_t(C) * F) return;
    const int c = int(w / F), f = int(w - int64_t(c) * F);
    const int64_t a = class_off[c], n = class_off[c + 1] - a;
    const T *row = mid + int64_t(f) * m_stride;
    const int64_t *ix = col + a;
    const hmm::ClassStats s = hmm::class_stats([&](int64_t i) { return double(row[ix[i]]); }, n, F == 1);
    const int64_t cf = int64_t(C) * F;
    out[w] = s.sum;
    out[cf + w] = s.mean;
    out[2 * cf + w] = s.ssq;
    out[3 * cf + w] = s.std;
}

// One thread per (clip, window, state), consecutive threads on consecutive windows of one (clip, state): e[row, state] of the
// slice, row = the clip's first row + window.  clips[2b] = the clip's window count, clips[2b + 1] its first global row.
// A non-finite feature of a valid window raises bad[b].  kWindowMajor: clip b is a C-contiguous [m_stride, F] matrix whose
// rows NumPy sums pairwise; else [F, m_stride], summed in sequence unless the clip has one window.
template <class T, bool kWindowMajor>
__global__ void __launch_bounds__(128) hmm_emission_kernel(const T *__restrict__ mid, int F, int64_t m_stride,
                                                           const int64_t *__restrict__ clips, int64_t b0, int64_t row_base,
                                                           int C, const double *__restrict__ mu, const double *__restrict__ var,
                                                           const double *__restrict__ konst, double *__restrict__ e,
                                                           int32_t *__restrict__ bad)
{
    const int64_t b = b0 + blockIdx.z;
    const int j = blockIdx.y;
    const int64_t t = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    const int64_t n = clips[2 * b];
    if (t >= n) return;
    const int64_t f_stride = kWindowMajor ? 1 : m_stride;
    const T *x = mid + size_t(b) * F * m_stride + (kWindowMajor ? t * F : t);
    auto xf = [&](int64_t f) { return double(x[f * f_stride]); };
    if (j == 0) {
        bool finite = true;
        for (int f = 0; f < F; ++f) finite &= isfinite(x[int64_t(f) * f_stride]);
        if (!finite) bad[b] = 1;
    }
    e[(clips[2 * b + 1] - row_base + t) * C + j] =
        hmm::emission(xf, mu + size_t(j) * F, var + size_t(j) * F, F, konst[j], kWindowMajor || n == 1);
}

// One warp per clip: the forward pass serial in t, lanes on states j, j + 32, ...; delta_{t-1} and delta_t in shared memory,
// the backpointers in the slice's scratch; then lane 0 backtracks.  ids[b, t] for t < n, zero up to m_stride; a refused clip
// (bad[b]) is not written.
__global__ void __launch_bounds__(32) hmm_viterbi_kernel(const int64_t *__restrict__ clips, int64_t b0, int64_t row_base, int C,
                                                         int64_t m_stride, const double *__restrict__ log_start,
                                                         const double *__restrict__ log_trans, const double *__restrict__ e,
                                                         int32_t *__restrict__ bp, const int32_t *__restrict__ bad,
                                                         int32_t *__restrict__ ids)
{
    extern __shared__ double delta[];
    const int64_t b = b0 + blockIdx.x;
    if (bad[b]) return;
    const int64_t n = clips[2 * b], r0 = clips[2 * b + 1] - row_base;
    const int lane = threadIdx.x;
    const double *eb = e + r0 * C;
    int32_t *bpb = bp + r0 * C;
    double *cur = delta, *prev = delta + C;
    for (int j = lane; j < C; j += 32) cur[j] = hmm::dadd(log_start[j], eb[j]);
    for (int64_t t = 1; t < n; ++t) {
        double *tmp = prev;
        prev = cur;
        cur = tmp;
        __syncwarp();
        for (int j = lane; j < C; j += 32) {
            int32_t p;
            cur[j] = hmm::step([prev](int32_t i) { return prev[i]; }, [log_trans, C, j](int32_t i) { return log_trans[int64_t(i) * C + j]; },
                               C, eb[t * C + j], p);
            bpb[t * C + j] = p;
        }
    }
    __syncwarp();
    int32_t *out = ids + size_t(b) * m_stride;
    if (lane == 0) {
        int32_t s = hmm::last_state([cur](int32_t i) { return cur[i]; }, C);
        out[n - 1] = s;
        for (int64_t t = n - 1; t > 0; --t) {
            s = bpb[t * C + s];
            out[t - 1] = s;
        }
    }
    for (int64_t t = n + lane; t < m_stride; t += 32) out[t] = 0;
}

namespace {
bool hmm_counts_ok(const int64_t *h_n, int64_t n_clips, int64_t m_stride, int64_t lo)
{
    for (int64_t b = 0; b < n_clips; ++b)
        if (h_n[b] < lo || h_n[b] > m_stride) return false;
    return true;
}
}  // namespace

extern "C" int b200aa_hmm_statistics(const void *d_mid, int dtype, int64_t n_clips, int n_feats, int64_t m_stride,
                                     const int64_t *h_n_windows, int n_classes, const int64_t *h_class_off,
                                     const int64_t *h_idx, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_hmm_statistics");
    REFUSE_CAPTURE(stream, "b200aa_hmm_statistics", kWhyHostArrays);
    if (!d_mid || !h_n_windows || !h_class_off || !h_idx || !d_out || n_clips < 1 || n_feats < 1 || m_stride < 1 ||
        n_classes < 1 || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64) || h_class_off[0] != 0 ||
        !hmm_counts_ok(h_n_windows, n_clips, m_stride, 0))
        return B200AA_ERR_INVALID;
    std::vector<int64_t> first(size_t(n_clips) + 1, 0);              // first concatenated window of each clip
    for (int64_t b = 0; b < n_clips; ++b) first[b + 1] = first[b] + h_n_windows[b];
    for (int c = 0; c < n_classes; ++c)
        if (h_class_off[c + 1] < h_class_off[c]) return B200AA_ERR_INVALID;
    const int64_t n_idx = h_class_off[n_classes];
    // [class offsets | element offset of each listed window's feature 0]
    std::vector<int64_t> head(size_t(n_classes) + 1 + size_t(n_idx));
    std::memcpy(head.data(), h_class_off, (size_t(n_classes) + 1) * sizeof(int64_t));
    for (int64_t i = 0; i < n_idx; ++i) {
        const int64_t g = h_idx[i];
        if (g < 0 || g >= first[n_clips]) return B200AA_ERR_INVALID;
        const int64_t b = int64_t(std::upper_bound(first.begin(), first.end(), g) - first.begin()) - 1;
        head[n_classes + 1 + i] = b * n_feats * m_stride + (g - first[b]);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(head.size() * sizeof(int64_t));
    if (rc != B200AA_OK) return rc;
    int64_t *d_head = static_cast<int64_t *>(scratch.get());
    CK(cudaMemcpyAsync(d_head, head.data(), head.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const int64_t threads = int64_t(n_classes) * n_feats;
    const unsigned blocks = unsigned((threads + 127) / 128);
    with_real_type(dtype, [&](auto t) {
        hmm_stats_kernel<<<blocks, 128, 0, st>>>(static_cast<const decltype(t) *>(d_mid), n_feats, m_stride, d_head + n_classes + 1,
                                                 d_head, n_classes, d_out);
    });
    CK_LAUNCH("hmm_stats_kernel");
    return scratch.done(B200AA_OK);
}

namespace {
// b200aa_hmm_decode / b200aa_hmm_decode_f64 after their argument checks
template <class T, bool kWindowMajor>
int hmm_decode(const T *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, const int64_t *h_n_windows, int n_states,
               const double *d_log_start, const double *d_log_trans, const double *d_means, const double *d_vars,
               const double *d_const, int32_t *d_ids, int32_t *d_bad, void *stream)
{
    // per clip (window count, first global row); slices of whole clips whose e + backpointers stay under kScratchSliceBytes
    // (a clip larger than that on its own is a slice of its own), at most 65535 clips (grid z)
    const size_t row_bytes = size_t(n_states) * (sizeof(double) + sizeof(int32_t));
    std::vector<int64_t> clips(2 * size_t(n_clips));
    std::vector<int64_t> cuts{0};
    int64_t rows = 0, slice_rows = 0, max_rows = 0;
    for (int64_t b = 0; b < n_clips; ++b) {
        const int64_t n = h_n_windows[b];
        if (b > cuts.back() && ((slice_rows + n) * row_bytes > kScratchSliceBytes || b - cuts.back() == 65535)) {
            cuts.push_back(b);
            slice_rows = 0;
        }
        clips[2 * b] = n;
        clips[2 * b + 1] = rows;
        rows += n;
        slice_rows += n;
        max_rows = std::max(max_rows, slice_rows);
    }
    cuts.push_back(n_clips);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = 2 * size_t(n_states) * sizeof(double);
    Layout L;
    const size_t clips_at = L.add(clips.size() * sizeof(int64_t)), e_at = L.add(size_t(max_rows) * n_states * sizeof(double)),
                 bp_at = L.add(size_t(max_rows) * n_states * sizeof(int32_t));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(L.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const int64_t *d_clips = Layout::at<const int64_t>(base, clips_at);
    double *e = Layout::at<double>(base, e_at);
    int32_t *bp = Layout::at<int32_t>(base, bp_at);
    CK(cudaMemcpyAsync(base, clips.data(), clips.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_bad, 0, size_t(n_clips) * sizeof(int32_t), st));
    for (size_t s = 0; s + 1 < cuts.size(); ++s) {
        const int64_t b0 = cuts[s], b1 = cuts[s + 1];
        int64_t max_n = 0;
        for (int64_t b = b0; b < b1; ++b) max_n = std::max(max_n, h_n_windows[b]);
        const int64_t row_base = clips[2 * b0 + 1];
        hmm_emission_kernel<T, kWindowMajor><<<dim3(unsigned((max_n + 127) / 128), unsigned(n_states), unsigned(b1 - b0)), 128, 0,
                                               st>>>(d_mid, n_feats, m_stride, d_clips, b0, row_base, n_states, d_means, d_vars,
                                                     d_const, e, d_bad);
        CK_LAUNCH("hmm_emission_kernel");
        hmm_viterbi_kernel<<<unsigned(b1 - b0), 32, smem, st>>>(d_clips, b0, row_base, n_states, m_stride, d_log_start,
                                                               d_log_trans, e, bp, d_bad, d_ids);
        CK_LAUNCH("hmm_viterbi_kernel");
    }
    return scratch.done(B200AA_OK);
}

bool hmm_decode_ok(const void *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, const int64_t *h_n_windows, int n_states,
                   const double *d_log_start, const double *d_log_trans, const double *d_means, const double *d_vars,
                   const double *d_const, int32_t *d_ids, int32_t *d_bad)
{
    return d_mid && h_n_windows && d_log_start && d_log_trans && d_means && d_vars && d_const && d_ids && d_bad && n_clips >= 1 &&
           n_feats >= 1 && m_stride >= 1 && n_states >= 1 && n_states <= hmm::kMaxStates &&
           hmm_counts_ok(h_n_windows, n_clips, m_stride, 1);
}
}  // namespace

extern "C" int b200aa_hmm_decode(const float *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, const int64_t *h_n_windows,
                                 int n_states, const double *d_log_start, const double *d_log_trans, const double *d_means,
                                 const double *d_vars, const double *d_const, int32_t *d_ids, int32_t *d_bad, void *stream)
{
    NvtxRange nvtx_("b200aa_hmm_decode");
    REFUSE_CAPTURE(stream, "b200aa_hmm_decode", kWhyHostArrays);
    if (!hmm_decode_ok(d_mid, n_clips, n_feats, m_stride, h_n_windows, n_states, d_log_start, d_log_trans, d_means, d_vars,
                       d_const, d_ids, d_bad))
        return B200AA_ERR_INVALID;
    return hmm_decode<float, false>(d_mid, n_clips, n_feats, m_stride, h_n_windows, n_states, d_log_start, d_log_trans, d_means,
                                    d_vars, d_const, d_ids, d_bad, stream);
}

extern "C" int b200aa_hmm_decode_f64(const double *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, int window_major,
                                     const int64_t *h_n_windows, int n_states, const double *d_log_start,
                                     const double *d_log_trans, const double *d_means, const double *d_vars,
                                     const double *d_const, int32_t *d_ids, int32_t *d_bad, void *stream)
{
    NvtxRange nvtx_("b200aa_hmm_decode_f64");
    REFUSE_CAPTURE(stream, "b200aa_hmm_decode_f64", kWhyHostArrays);
    if ((window_major != 0 && window_major != 1) ||
        !hmm_decode_ok(d_mid, n_clips, n_feats, m_stride, h_n_windows, n_states, d_log_start, d_log_trans, d_means, d_vars,
                       d_const, d_ids, d_bad))
        return B200AA_ERR_INVALID;
    auto run = window_major ? hmm_decode<double, true> : hmm_decode<double, false>;
    return run(d_mid, n_clips, n_feats, m_stride, h_n_windows, n_states, d_log_start, d_log_trans, d_means, d_vars, d_const,
               d_ids, d_bad, stream);
}
