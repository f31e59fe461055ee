// libb200aa.so -- kNN classification and its cross-validation (kernels 5 and 6).
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/b200aa.h"
#include "entry.h"
#include "knn.cuh"
#include "knn_cv.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernels 5 and 6: kNN classification (audioTrainTest.py:33-49), bit for bit the reference's Knn.classify per query
// (csrc/knn.cuh), and its cross-validation (audioTrainTest.py:576-771, csrc/knn_cv.cuh)
// ------------------------------------------------------------------------------------------------
// The distance and select kernels run a batch of problems (knn::Problem): `probs` on the device, one problem per grid z
// (distance) or y (select).  Kernel 5 passes NULL and its one problem by value in `one`.
//
// keys[q][i] = key_of(distance(query q, training row i)) for a 64-query x 64-row tile per CTA.  Both tiles are staged
// 16 features at a time, transposed to [feature][row]; each thread runs 4 x 4 independent chains (queries ty + 16a,
// rows tx + 16b), so the 136-long dependent DADD chain of one pair is hidden behind 15 others.
template <class Tq>
__global__ void __launch_bounds__(knn::kThreads, 3) knn_dist_kernel(const knn::Problem *__restrict__ probs, knn::Problem one,
                                                                 const double *__restrict__ feats, int F,
                                                                 const Tq *__restrict__ q, int64_t q_stride,
                                                                 uint64_t *__restrict__ keys)
{
    static_assert(knn::kQ == knn::kT && knn::kQ == 64 && knn::kThreads == 256, "tile shape");
    __shared__ double sq[knn::kF][knn::kQ + 1];
    __shared__ double sv[knn::kF][knn::kT + 1];
    const knn::Problem pb = probs ? probs[blockIdx.z] : one;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t t0 = int64_t(blockIdx.x) * knn::kT;
    const int64_t q0 = int64_t(blockIdx.y) * knn::kQ;
    const int64_t N = pb.N, n_slice = pb.n_q;
    if (t0 >= N || q0 >= n_slice) return;       // a tile past this problem: the grid covers the batch's largest
    feats += pb.train0 * F;
    q += pb.q0 * q_stride;
    keys += pb.key0;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int f0 = 0; f0 < F; f0 += knn::kF) {
        const int nf = min(knn::kF, F - f0);
        __syncthreads();
        for (int e = threadIdx.x; e < knn::kQ * knn::kF; e += knn::kThreads) {
            const int r = e / knn::kF, j = e % knn::kF;
            const int64_t qi = q0 + r, ti = t0 + r;
            sq[j][r] = (j < nf && qi < n_slice) ? double(q[qi * q_stride + f0 + j]) : 0.0;      // float32: widened exactly
            sv[j][r] = (j < nf && ti < N) ? feats[ti * F + f0 + j] : 0.0;
        }
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < nf; ++j) {
            double x[4], v[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) x[a] = sq[j][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 4; ++b) v[b] = sv[j][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = knn::dist_step(acc[a][b], x[a], v[b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int64_t qi = q0 + ty + 16 * a;
        if (qi >= n_slice) continue;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int64_t ti = t0 + tx + 16 * b;
            if (ti < N) keys[qi * N + ti] = knn::key_of(knn::dsqrt(acc[a][b]));
        }
    }
}

// One CTA per query: the k-th smallest key by radix select (8 passes of 256 bins over the keys sharing the prefix found so
// far), then one pass in training-index order that selects the keys below it and the first r equal to it, counting the
// selected entries' classes in shared memory, kVoteClasses classes per pass.  Kernel 5 (kCounts false) writes P[q][0..C)
// and the first maximum as ids[q]; kernel 6 writes the first maximum as pred[q] and counts it in the problem's confusion
// block, counts[id][truth][pred] (integer atomics: the counts do not depend on the order).
struct KnnVotes {
    int64_t *ids;
    double *P;
    int32_t *pred;
    const int32_t *truth;               // kernel 6: the class of each query row; outside [0, n_classes) it is not counted
    unsigned long long *counts;
    int n_classes;
};

template <bool kCounts>
__global__ void __launch_bounds__(knn::kThreads) knn_select_kernel(const knn::Problem *__restrict__ probs, knn::Problem one,
                                                                   const uint64_t *__restrict__ keys,
                                                                   const int32_t *__restrict__ slots, KnnVotes out)
{
    constexpr int kWarps = knn::kThreads / 32;
    __shared__ unsigned hist[knn::kBins];
    __shared__ unsigned votes[knn::kVoteClasses];
    __shared__ unsigned warp_eq[kWarps];
    __shared__ int64_t warp_best_c[kWarps], warp_best_i[kWarps];
    __shared__ uint64_t s_prefix;
    __shared__ int64_t s_rank;
    const knn::Problem pb = probs ? probs[blockIdx.y] : one;
    if (blockIdx.x >= pb.n_q) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t N = pb.N, k = pb.k;
    const int C = pb.C;
    const int64_t q = pb.out0 + blockIdx.x;
    const uint64_t *row = keys + pb.key0 + int64_t(blockIdx.x) * N;
    slots += pb.train0;

    uint64_t thr = knn::kAll;           // k >= N: every entry is selected
    int64_t r = 0;
    if (k < N) {
        uint64_t prefix = 0;
        int64_t rank = k;
        for (int shift = 64 - knn::kDigitBits; shift >= 0; shift -= knn::kDigitBits) {
            const uint64_t mask = knn::prefix_mask(shift);
            for (int b = tid; b < knn::kBins; b += knn::kThreads) hist[b] = 0;
            __syncthreads();
            for (int64_t i = tid; i < N; i += knn::kThreads) {
                const uint64_t key = row[i];
                if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & (knn::kBins - 1)], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                const int d = knn::select_digit(hist, rank);
                s_prefix = prefix | (uint64_t(d) << shift);
                s_rank = rank;
            }
            __syncthreads();
            prefix = s_prefix;
            rank = s_rank;
        }
        thr = prefix;
        r = rank;
    }

    int64_t best_c = -1, best_i = 0;    // thread 0: the first maximum over the classes done so far
    for (int c0 = 0; c0 < C; c0 += knn::kVoteClasses) {
        const int nc = min(knn::kVoteClasses, C - c0);
        for (int c = tid; c < knn::kVoteClasses; c += knn::kThreads) votes[c] = 0;
        __syncthreads();
        int64_t eq_done = 0;            // keys equal to thr at indices below this chunk
        for (int64_t base = 0; base < N; base += knn::kThreads) {
            const int64_t i = base + tid;
            const uint64_t key = i < N ? row[i] : 0;
            const bool eq = i < N && key == thr;
            const unsigned m = __ballot_sync(0xffffffffu, eq);
            if (lane == 0) warp_eq[warp] = __popc(m);
            __syncthreads();
            int64_t before = eq_done + __popc(m & ((1u << lane) - 1u)), total = 0;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) {
                if (w < warp) before += warp_eq[w];
                total += warp_eq[w];
            }
            if (i < N && knn::selected(key, thr, before, r)) {
                const int s = slots[i];
                if (s >= c0 && s < c0 + nc) atomicAdd(&votes[s - c0], 1u);
            }
            eq_done += total;
            __syncthreads();
        }
        int64_t bc = -1, bi = 0;
        for (int c = tid; c < nc; c += knn::kThreads) {
            if (!kCounts) out.P[q * C + c0 + c] = knn::vote(votes[c], k);
            if (bc < 0 || knn::better(votes[c], c0 + c, bc, bi)) { bc = votes[c]; bi = c0 + c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int64_t oc = __shfl_xor_sync(0xffffffffu, bc, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oc >= 0 && (bc < 0 || knn::better(oc, oi, bc, bi))) { bc = oc; bi = oi; }
        }
        if (lane == 0) { warp_best_c[warp] = bc; warp_best_i[warp] = bi; }
        __syncthreads();
        if (tid == 0)
            for (int w = 0; w < kWarps; ++w)
                if (warp_best_c[w] >= 0 && (best_c < 0 || knn::better(warp_best_c[w], warp_best_i[w], best_c, best_i))) {
                    best_c = warp_best_c[w];
                    best_i = warp_best_i[w];
                }
        __syncthreads();
    }
    if (tid == 0) {
        if (kCounts) {
            out.pred[q] = int32_t(best_i);
            const int32_t t = out.truth[pb.q0 + blockIdx.x];
            if (t >= 0 && t < out.n_classes)
                atomicAdd(&out.counts[(int64_t(pb.id) * out.n_classes + t) * out.n_classes + best_i], 1ull);
        } else {
            out.ids[q] = best_i;
        }
    }
}

extern "C" int b200aa_knn_classify(const double *d_feats, const int32_t *d_slots, int64_t n_train, int n_feats, int n_classes,
                                   int64_t k, const void *d_query, int dtype, int64_t n_query, int64_t q_stride, int64_t *d_ids,
                                   double *d_P, void *stream)
{
    NvtxRange nvtx_("b200aa_knn_classify");
    REFUSE_CAPTURE(stream, "b200aa_knn_classify", kWhyHostArrays);
    if (!d_feats || !d_slots || !d_query || !d_ids || !d_P || n_train < 1 || n_train > INT32_MAX || n_feats < 1 ||
        n_classes < 1 || k < 1 || n_query < 0 || q_stride < n_feats || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (n_query == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // scratch: one key per (query, training row); queries go in slices whose keys stay below 256 MiB
    const size_t row_bytes = size_t(n_train) * sizeof(uint64_t);
    const int64_t slice = std::max<int64_t>(1, std::min<int64_t>({n_query, int64_t(kScratchSliceBytes / row_bytes),
                                                                   int64_t(65535) * knn::kQ}));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(size_t(slice) * row_bytes);
    if (rc != B200AA_OK) return rc;
    uint64_t *keys = static_cast<uint64_t *>(scratch.get());
    for (int64_t q0 = 0; q0 < n_query; q0 += slice) {
        const int64_t ns = std::min<int64_t>(slice, n_query - q0);
        const knn::Problem one{0, n_train, 0, ns, 0, q0, k, 0, 0, n_classes, 0};
        const dim3 grid((unsigned)((n_train + knn::kT - 1) / knn::kT), (unsigned)((ns + knn::kQ - 1) / knn::kQ));
        with_real_type(dtype, [&](auto t) {
            knn_dist_kernel<<<grid, knn::kThreads, 0, st>>>(nullptr, one, d_feats, n_feats,
                                                            static_cast<const decltype(t) *>(d_query) + q0 * q_stride, q_stride, keys);
        });
        CK_LAUNCH("knn_dist_kernel");
        KnnVotes out{};
        out.ids = d_ids;
        out.P = d_P;
        knn_select_kernel<false><<<(unsigned)ns, knn::kThreads, 0, st>>>(nullptr, one, keys, d_slots, out);
        CK_LAUNCH("knn_select_kernel");
    }
    return scratch.done(B200AA_OK);
}

// Kernel 6, first step of a slice: per (problem, column) StandardScaler().fit over the problem's training rows in the
// split's order, then its training and query rows standardised into the slice's matrices, the training rows' slots and
// the query rows' classes.  One thread per column: each fit is a sequential chain, as scikit-learn sums it.
__global__ void __launch_bounds__(knn::kFitThreads) knn_cv_gather_kernel(const knn::Problem *__restrict__ probs,
                                                                         const double *__restrict__ X, const int32_t *__restrict__ y,
                                                                         int F, const int32_t *__restrict__ train_idx,
                                                                         const int32_t *__restrict__ test_idx,
                                                                         double *__restrict__ train, double *__restrict__ query,
                                                                         int32_t *__restrict__ slots, int32_t *__restrict__ truth)
{
    const knn::Problem pb = probs[blockIdx.y];
    const int32_t *tr = train_idx + pb.src_train, *te = test_idx + pb.src_test;
    if (blockIdx.x == 0) {
        for (int64_t i = threadIdx.x; i < pb.N; i += knn::kFitThreads) slots[pb.train0 + i] = knn::split_slot(y[tr[i]], pb.C);
        for (int64_t i = threadIdx.x; i < pb.n_q; i += knn::kFitThreads) truth[pb.q0 + i] = y[te[i]];
    }
    const int j = blockIdx.x * knn::kFitThreads + threadIdx.x;
    if (j >= F) return;
    const knn::Scale s = knn::scaler_fit([&](int64_t i) { return X[int64_t(tr[i]) * F + j]; }, pb.N);
    for (int64_t i = 0; i < pb.N; ++i) train[(pb.train0 + i) * F + j] = knn::standardise(X[int64_t(tr[i]) * F + j], s);
    for (int64_t i = 0; i < pb.n_q; ++i) query[(pb.q0 + i) * F + j] = knn::standardise(X[int64_t(te[i]) * F + j], s);
}

// The host half of kernel 6: validates the splits, cuts them into work items (a problem, or a range of its test rows when
// one problem's scratch passes the bound) and packs the items into slices whose scratch stays under kScratchSliceBytes.
namespace {
constexpr int64_t kMaxItems = 65535;    // grid z of the distance kernel, grid y of the select kernel

struct CvSlice {
    int64_t first, end;                 // items [first, end)
    int64_t train_rows, query_rows, keys, max_N, max_q;
};
}  // namespace

extern "C" int b200aa_knn_cross_validate(const double *d_X, const int32_t *d_y, int64_t n, int n_feats, int n_classes,
                                         int64_t n_problems, const int64_t *h_train_off, const int32_t *h_train_idx,
                                         const int64_t *h_test_off, const int32_t *h_test_idx, const int64_t *h_k,
                                         const int32_t *h_classes, int32_t *d_pred, int64_t *d_counts, void *stream)
{
    NvtxRange nvtx_("b200aa_knn_cross_validate");
    REFUSE_CAPTURE(stream, "b200aa_knn_cross_validate", kWhyHostArrays);
    if (!d_X || !d_y || !h_train_off || !h_train_idx || !h_test_off || !h_test_idx || !h_k || !h_classes || !d_pred ||
        !d_counts || n < 1 || n > INT32_MAX || n_feats < 1 || n_classes < 1 || n_problems < 0 || h_train_off[0] != 0 ||
        h_test_off[0] != 0)
        return B200AA_ERR_INVALID;
    for (int64_t p = 0; p < n_problems; ++p)
        if (h_train_off[p + 1] - h_train_off[p] < 1 || h_test_off[p + 1] - h_test_off[p] < 1 || h_k[p] < 1 ||
            h_classes[p] < 1 || h_classes[p] > n_classes)
            return B200AA_ERR_INVALID;
    const int64_t n_train_all = h_train_off[n_problems], n_test_all = h_test_off[n_problems];
    for (int64_t i = 0; i < n_train_all; ++i)
        if (h_train_idx[i] < 0 || h_train_idx[i] >= n) return B200AA_ERR_INVALID;
    for (int64_t i = 0; i < n_test_all; ++i)
        if (h_test_idx[i] < 0 || h_test_idx[i] >= n) return B200AA_ERR_INVALID;
    if (n_problems == 0) return B200AA_OK;

    // work items and slices: per item its standardised rows, slots / classes and keys
    const size_t row = size_t(n_feats) * sizeof(double) + sizeof(int32_t);
    std::vector<knn::Problem> items;
    std::vector<CvSlice> slices;
    CvSlice cur{0, 0, 0, 0, 0, 0, 0};
    size_t cur_bytes = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t N = h_train_off[p + 1] - h_train_off[p], T = h_test_off[p + 1] - h_test_off[p];
        const size_t fixed = size_t(N) * row, per_q = row + size_t(N) * sizeof(uint64_t);
        const int64_t fit = fixed < kScratchSliceBytes ? int64_t((kScratchSliceBytes - fixed) / per_q) : 0;
        const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>({T, fit, int64_t(65535) * knn::kQ}));
        for (int64_t a = 0; a < T; a += chunk) {
            const int64_t nq = std::min(chunk, T - a);
            const size_t bytes = fixed + size_t(nq) * per_q;
            if (cur.end > cur.first && (cur_bytes + bytes > kScratchSliceBytes || cur.end - cur.first == kMaxItems)) {
                slices.push_back(cur);
                cur = CvSlice{cur.end, cur.end, 0, 0, 0, 0, 0};
                cur_bytes = 0;
            }
            items.push_back(knn::Problem{cur.train_rows, N, cur.query_rows, nq, cur.keys, h_test_off[p] + a, h_k[p],
                                         h_train_off[p], h_test_off[p] + a, h_classes[p], int32_t(p)});
            cur.end++;
            cur.train_rows += N;
            cur.query_rows += nq;
            cur.keys += N * nq;
            cur.max_N = std::max(cur.max_N, N);
            cur.max_q = std::max(cur.max_q, nq);
            cur_bytes += bytes;
        }
    }
    slices.push_back(cur);

    // the items and the training and test indices, uploaded once as one head
    Layout L;
    const size_t items_at = L.add(items.size() * sizeof(knn::Problem)), tr_at = L.add(size_t(n_train_all) * sizeof(int32_t)),
                 te_at = L.add(size_t(n_test_all) * sizeof(int32_t));
    std::vector<char> head(te_at + size_t(n_test_all) * sizeof(int32_t));
    std::memcpy(head.data() + items_at, items.data(), items.size() * sizeof(knn::Problem));
    std::memcpy(head.data() + tr_at, h_train_idx, size_t(n_train_all) * sizeof(int32_t));
    std::memcpy(head.data() + te_at, h_test_idx, size_t(n_test_all) * sizeof(int32_t));
    // then one slice's matrices, slots, classes and keys, each sized by the largest slice
    int64_t train_rows = 0, query_rows = 0, n_keys = 0;
    for (const CvSlice &s : slices) {
        train_rows = std::max(train_rows, s.train_rows);
        query_rows = std::max(query_rows, s.query_rows);
        n_keys = std::max(n_keys, s.keys);
    }
    const size_t train_at = L.add(size_t(train_rows) * n_feats * sizeof(double)),
                 query_at = L.add(size_t(query_rows) * n_feats * sizeof(double)),
                 slots_at = L.add(size_t(train_rows) * sizeof(int32_t)), truth_at = L.add(size_t(query_rows) * sizeof(int32_t)),
                 keys_at = L.add(size_t(n_keys) * sizeof(uint64_t));

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(L.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const knn::Problem *d_items = Layout::at<const knn::Problem>(base, items_at);
    const int32_t *d_tr = Layout::at<const int32_t>(base, tr_at), *d_te = Layout::at<const int32_t>(base, te_at);
    double *train = Layout::at<double>(base, train_at), *query = Layout::at<double>(base, query_at);
    int32_t *slots = Layout::at<int32_t>(base, slots_at), *truth = Layout::at<int32_t>(base, truth_at);
    uint64_t *keys = Layout::at<uint64_t>(base, keys_at);
    CK(cudaMemcpyAsync(base, head.data(), head.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_counts, 0, size_t(n_problems) * n_classes * n_classes * sizeof(int64_t), st));

    KnnVotes out{};
    out.pred = d_pred;
    out.truth = truth;
    out.counts = reinterpret_cast<unsigned long long *>(d_counts);
    out.n_classes = n_classes;
    const knn::Problem none{};
    for (const CvSlice &s : slices) {
        const unsigned n_items = unsigned(s.end - s.first);
        const knn::Problem *probs = d_items + s.first;
        knn_cv_gather_kernel<<<dim3((n_feats + knn::kFitThreads - 1) / knn::kFitThreads, n_items), knn::kFitThreads, 0, st>>>(
            probs, d_X, d_y, n_feats, d_tr, d_te, train, query, slots, truth);
        CK_LAUNCH("knn_cv_gather_kernel");
        const dim3 grid((unsigned)((s.max_N + knn::kT - 1) / knn::kT), (unsigned)((s.max_q + knn::kQ - 1) / knn::kQ), n_items);
        knn_dist_kernel<<<grid, knn::kThreads, 0, st>>>(probs, none, train, n_feats, static_cast<const double *>(query),
                                                        int64_t(n_feats), keys);
        CK_LAUNCH("knn_dist_kernel");
        knn_select_kernel<true><<<dim3((unsigned)s.max_q, n_items), knn::kThreads, 0, st>>>(probs, none, keys, slots, out);
        CK_LAUNCH("knn_select_kernel");
    }
    return scratch.done(B200AA_OK);
}
