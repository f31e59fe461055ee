// libb200aa.so -- scaler, outlier rule and per-frame pooling (kernel 11).
#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

#include "../../include/b200aa.h"
#include "cluster.cuh"
#include "entry.h"
#include "front.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// kernel 11: StandardScaler().fit_transform, the feature-outlier rule and the LDA branch's pooling of speaker_diarization
// and music_thumbnailing (audioSegmentation.py:51-52, :858-906), bit for bit (csrc/front.cuh)
// ------------------------------------------------------------------------------------------------
// One thread per (matrix, column): the column's fit, and the matrix's flag when it holds +-inf.  blockIdx.y strides over
// the matrices.
template <class T>
__global__ void __launch_bounds__(128) front_fit_kernel(const T *__restrict__ X, int64_t mat_stride, int64_t row_stride,
                                                        int64_t col_stride, const int64_t *__restrict__ rows, int64_t n_mats,
                                                        int D, bool pairwise, double *__restrict__ mean,
                                                        double *__restrict__ scale, int32_t *__restrict__ bad)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= D) return;
    for (int64_t b = blockIdx.y; b < n_mats; b += gridDim.y) {
        const T *x = X + b * mat_stride + j * col_stride;
        bool inf;
        const knn::Scale s = front::scaler_fit([x, row_stride](int64_t i) { return double(x[i * row_stride]); }, rows[b],
                                               pairwise, inf);
        mean[b * D + j] = s.mean;
        scale[b * D + j] = s.scale;
        if (inf) bad[b] = 1;
    }
}

// (x - mean) / scale of every entry: blockIdx.y strides over the matrices, x over the entries of one, in the order of the
// input's smaller stride
template <class T>
__global__ void __launch_bounds__(256) front_transform_kernel(const T *__restrict__ X, int64_t mat_stride, int64_t row_stride,
                                                              int64_t col_stride, const int64_t *__restrict__ rows,
                                                              int64_t n_mats, int D, bool column_major,
                                                              const double *__restrict__ mean,
                                                              const double *__restrict__ scale, double *__restrict__ out,
                                                              const int64_t *__restrict__ out_off, int64_t out_row_stride,
                                                              int64_t out_col_stride)
{
    for (int64_t b = blockIdx.y; b < n_mats; b += gridDim.y) {
        const int64_t n = rows[b];
        for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < n * D; e += int64_t(gridDim.x) * blockDim.x) {
            const int64_t i = column_major ? e % n : e / D, j = column_major ? e / n : e % D;
            const knn::Scale s{mean[b * D + j], scale[b * D + j]};
            out[out_off[b] + i * out_row_stride + j * out_col_stride] =
                knn::standardise(double(X[b * mat_stride + i * row_stride + j * col_stride]), s);
        }
    }
}

extern "C" int b200aa_standard_scale(const void *d_X, int dtype, int64_t n_mats, int n_feats, const int64_t *h_rows,
                                     int64_t mat_stride, int64_t row_stride, int64_t col_stride, double *d_out,
                                     const int64_t *h_out_off, int64_t out_row_stride, int64_t out_col_stride,
                                     double *d_mean, double *d_scale, int32_t *d_bad, void *stream)
{
    NvtxRange nvtx_("b200aa_standard_scale");
    REFUSE_CAPTURE(stream, "b200aa_standard_scale", "kernel 11 is not captured; call it eagerly");
    const int D = n_feats;
    if (!d_X || !h_rows || !d_out || !h_out_off || !d_mean || !d_scale || !d_bad || n_mats < 1 || D < 1 ||
        mat_stride < 0 || row_stride < 1 || col_stride < 1 || out_row_stride < 1 || out_col_stride < 1 ||
        (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    int64_t n_max = 0;
    for (int64_t b = 0; b < n_mats; ++b) {
        if (h_rows[b] < 1 || h_out_off[b] < 0) return B200AA_ERR_INVALID;
        n_max = std::max(n_max, h_rows[b]);
    }
    // NumPy reduces over axis 0 along the axis of smaller stride: pairwise down each column of a column-major matrix
    const bool pairwise = D == 1 || row_stride < col_stride;
    Layout L;
    const size_t rows_at = L.add(size_t(n_mats) * sizeof(int64_t)), off_at = L.add(size_t(n_mats) * sizeof(int64_t));
    std::vector<char> head(L.bytes(), 0);
    std::memcpy(head.data() + rows_at, h_rows, size_t(n_mats) * sizeof(int64_t));
    std::memcpy(head.data() + off_at, h_out_off, size_t(n_mats) * sizeof(int64_t));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(head.size());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const int64_t *d_rows = Layout::at<const int64_t>(base, rows_at), *d_off = Layout::at<const int64_t>(base, off_at);
    CK(cudaMemcpyAsync(base, head.data(), head.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_bad, 0, size_t(n_mats) * sizeof(int32_t), st));
    const unsigned grid_y = unsigned(std::min<int64_t>(n_mats, 65535));
    const int rc2 = with_real_type(dtype, [&](auto zero) {
        using T = decltype(zero);
        const T *X = static_cast<const T *>(d_X);
        front_fit_kernel<T><<<dim3(unsigned((D + 127) / 128), grid_y), 128, 0, st>>>(
            X, mat_stride, row_stride, col_stride, d_rows, n_mats, D, pairwise, d_mean, d_scale, d_bad);
        CK_LAUNCH("front_fit_kernel");
        const unsigned grid_x = unsigned(std::min<int64_t>((n_max * D + 255) / 256, 4096));
        front_transform_kernel<T><<<dim3(grid_x, grid_y), 256, 0, st>>>(X, mat_stride, row_stride, col_stride, d_rows, n_mats,
                                                                       D, pairwise, d_mean, d_scale, d_out, d_off,
                                                                       out_row_stride, out_col_stride);
        CK_LAUNCH("front_transform_kernel");
        return int(B200AA_OK);
    });
    if (rc2 != B200AA_OK) return rc2;
    return scratch.done(B200AA_OK);
}

// One CTA: dist_all from the D x D distances (front::column_sum per column), then the threshold and the flags
__global__ void __launch_bounds__(front::kOutlierThreads) front_outlier_kernel(const double *__restrict__ dist, int D,
                                                                              double *__restrict__ dist_all,
                                                                              double *__restrict__ mean,
                                                                              unsigned char *__restrict__ keep)
{
    __shared__ double thr;
    for (int j = threadIdx.x; j < D; j += blockDim.x)
        dist_all[j] = front::column_sum([dist, D](int i, int c) { return dist[int64_t(i) * D + c]; }, D, j);
    __syncthreads();
    if (threadIdx.x == 0) {
        *mean = front::outlier_mean([dist_all](int64_t j) { return dist_all[j]; }, D);
        thr = front::outlier_threshold(*mean);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < D; j += blockDim.x) keep[j] = dist_all[j] < thr;
}

extern "C" int b200aa_outlier_columns(const double *d_X, int64_t n_rows, int n_feats, int64_t col_stride,
                                      double *d_dist_all, double *d_mean, unsigned char *d_keep, void *stream)
{
    NvtxRange nvtx_("b200aa_outlier_columns");
    REFUSE_CAPTURE(stream, "b200aa_outlier_columns", "kernel 11 is not captured; call it eagerly");
    const int D = n_feats;
    if (!d_X || !d_dist_all || !d_mean || !d_keep || n_rows < 1 || D < 1 || D > front::kMaxFeats || col_stride < n_rows ||
        col_stride > INT_MAX)
        return B200AA_ERR_INVALID;
    // the distances of every pair of columns as one kernel 9 block segment: item u is column u, its n_rows values the chain
    cluster::Segment seg{};
    seg.n_left = seg.n_right = D;
    seg.n_feat = n_rows;
    seg.len = int64_t(D) * D;
    seg.kind = cluster::kBlock;
    Layout L;
    const size_t seg_at = L.add(sizeof seg), dist_at = L.add(size_t(D) * D * sizeof(double));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(L.bytes());
    if (rc != B200AA_OK) return rc;
    void *base = scratch.get();
    const cluster::Segment *d_seg = Layout::at<const cluster::Segment>(base, seg_at);
    double *dist = Layout::at<double>(base, dist_at);
    CK(cudaMemcpyAsync(base, &seg, sizeof seg, cudaMemcpyHostToDevice, st));
    cluster_dist_kernel<<<unsigned(cluster::tiles_of(seg)), cluster::kThreads, 0, st>>>(d_seg, 0, 1, d_X, int(col_stride),
                                                                                       dist);
    CK_LAUNCH("cluster_dist_kernel");
    front_outlier_kernel<<<1, front::kOutlierThreads, 0, st>>>(dist, D, d_dist_all, d_mean, d_keep);
    CK_LAUNCH("front_outlier_kernel");
    return scratch.done(B200AA_OK);
}

// One thread per (clip, feature, frame): the window's mean and std (front::pool_window)
template <class T>
__global__ void __launch_bounds__(256) front_pool_kernel(const T *__restrict__ x, int64_t clip_stride, int64_t row_stride,
                                                         const int64_t *__restrict__ frames, int64_t n_clips, int F,
                                                         int64_t t_max, int64_t ratio, double *__restrict__ out,
                                                         int64_t out_stride)
{
    for (int64_t b = blockIdx.y; b < n_clips; b += gridDim.y) {
        const int64_t nt = frames[b];
        for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < F * t_max; e += int64_t(gridDim.x) * blockDim.x) {
            const int64_t f = e / t_max, i = e - f * t_max;
            if (i >= nt) continue;
            const T *w = x + b * clip_stride + f * row_stride + i;
            double mean, std;
            front::pool_window([w](int64_t k) { return double(w[k]); }, min(ratio, nt - i), mean, std);
            double *o = out + (b * 2 * F + f) * out_stride + i;
            o[0] = mean;
            o[F * out_stride] = std;
        }
    }
}

extern "C" int b200aa_pool_frames(const void *d_st, int dtype, int64_t n_clips, int n_feats, int64_t clip_stride,
                                  int64_t row_stride, const int64_t *h_frames, int64_t ratio, double *d_out,
                                  int64_t out_stride, void *stream)
{
    NvtxRange nvtx_("b200aa_pool_frames");
    REFUSE_CAPTURE(stream, "b200aa_pool_frames", "kernel 11 is not captured; call it eagerly");
    const int F = n_feats;
    if (!d_st || !h_frames || !d_out || n_clips < 1 || F < 1 || ratio < 1 || clip_stride < 0 || row_stride < 0 ||
        (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    int64_t t_max = 0;
    for (int64_t b = 0; b < n_clips; ++b) {
        if (h_frames[b] < 1 || h_frames[b] > out_stride) return B200AA_ERR_INVALID;
        t_max = std::max(t_max, h_frames[b]);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(size_t(n_clips) * sizeof(int64_t));
    if (rc != B200AA_OK) return rc;
    int64_t *d_frames = static_cast<int64_t *>(scratch.get());
    CK(cudaMemcpyAsync(d_frames, h_frames, size_t(n_clips) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const unsigned grid_x = unsigned(std::min<int64_t>((F * t_max + 255) / 256, 1 << 16));
    const unsigned grid_y = unsigned(std::min<int64_t>(n_clips, 65535));
    const int rc2 = with_real_type(dtype, [&](auto zero) {
        using T = decltype(zero);
        front_pool_kernel<T><<<dim3(grid_x, grid_y), 256, 0, st>>>(static_cast<const T *>(d_st), clip_stride, row_stride,
                                                                   d_frames, n_clips, F, t_max, ratio, d_out, out_stride);
        CK_LAUNCH("front_pool_kernel");
        return int(B200AA_OK);
    });
    if (rc2 != B200AA_OK) return rc2;
    return scratch.done(B200AA_OK);
}
