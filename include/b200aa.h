/*
 * b200aa.h -- C ABI of libb200aa.so, the H100 (sm_90a) short-term / mid-term audio
 * feature extractor that replaces pyAudioAnalysis' NumPy hot path.
 *
 * Boundary rules: extern "C", plain pointers and sizes, no C++ / torch types, no
 * exceptions.  Every function returns 0 (B200AA_OK) or a negative b200aa_status.
 * Pointers named d_* are device pointers of the current CUDA device, h_* are host
 * pointers; the caller owns every buffer.  `stream` is a cudaStream_t passed as
 * void* (NULL = default stream); device-pointer entry points are asynchronous on it.
 *
 * The reference has no FFI of its own: its boundary is four Python functions.  Each
 * entry point below names the reference code it replaces (paths relative to
 * pyAudioAnalysis/ in the reference tree).  INTEGRATION.md shows the ctypes stub a
 * maintainer of the reference would add.
 */
#ifndef B200AA_H_
#define B200AA_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200AA_ABI_VERSION 1

typedef enum b200aa_status {
    B200AA_OK = 0,
    B200AA_ERR_INVALID = -1,      /* bad argument (NULL pointer, window < 2, step < 1, ...)              */
    B200AA_ERR_TOO_SHORT = -2,    /* clip shorter than one window: the reference raises ValueError
                                     ("need at least one array to concatenate", ShortTermFeatures.py:684) */
    B200AA_ERR_CHROMA = -3,       /* semitone index >= num_fft: the reference's chroma else-branch
                                     (ShortTermFeatures.py:290-294) raises ValueError                     */
    B200AA_ERR_MEL_RANGE = -4,    /* mel filter edge beyond num_fft: the reference raises IndexError
                                     (ShortTermFeatures.py:230-231)                                       */
    B200AA_ERR_CUDA = -5,         /* a CUDA call failed; see b200aa_last_cuda_error()                     */
    B200AA_ERR_UNSUPPORTED = -6,  /* window too large for the on-chip transform buffers                  */
    B200AA_ERR_NO_DEVICE = -7,    /* no CUDA device / not an sm_90 device                                 */
    B200AA_ERR_CAPTURE = -8       /* the stream is capturing a CUDA graph and this call cannot be captured: make it once
                                     outside capture first, or call it eagerly; b200aa_last_cuda_error() names the entry
                                     point and the reason                                                 */
} b200aa_status;

/* sample formats of the clip buffer */
#define B200AA_DTYPE_I16 0        /* int16 PCM as scipy.io.wavfile.read returns it (audioBasicIO.py:99) */
#define B200AA_DTYPE_F32 1        /* float32 samples (any scale; the path is scale invariant)           */
#define B200AA_DTYPE_F64 2        /* float64 (the float64 feature path, b200aa_knn_classify's query vectors) */

#define B200AA_N_BASE 34          /* ShortTermFeatures.py:580-585 */
#define B200AA_N_MEL 40           /* ShortTermFeatures.py:191-192 */
#define B200AA_N_MFCC 13

/* Per-clip affine normalisation y = a*(x - m) + bp that reproduces `/2**15` + dc_normalize()
 * (ShortTermFeatures.py:567-570, :14-19), plus exact thresholds for sign(x - mean).  32 bytes. */
typedef struct b200aa_clip_norm {
    float a;        /* 1 / (max|x - mean| + 2^15 * 1e-10)                      */
    float bp;       /* a * (m - mean)                                          */
    float m;        /* value nearest to the clip mean that is exact in float   */
    float lo;       /* largest representable sample value <= mean, minus m    */
    float hi;       /* smallest representable sample value >= mean, minus m   */
    float rsv[3];   /* scratch used while the statistics are accumulated       */
} b200aa_clip_norm;

/* Per-clip normalisation of the float64 path: y = (x / 32768.0 - mean) / scale, bit for bit the reference's
 * `signal / 2**15` + dc_normalize() in NumPy float64.  16 bytes. */
typedef struct b200aa_clip_norm_f64 {
    double mean;    /* np.mean(x / 32768.0)                          */
    double scale;   /* np.abs(x / 32768.0 - mean).max() + 1e-10      */
} b200aa_clip_norm_f64;

typedef struct b200aa_plan b200aa_plan;   /* opaque: constant tables of one (fs, window, step) on one device */

/* ------------------------------------------------------------------ library ---------- */
int         b200aa_abi_version(void);
const char *b200aa_status_string(int status);
const char *b200aa_last_cuda_error(void);        /* thread-local text of the last CUDA failure or capture refusal */
int         b200aa_device_ok(void);              /* B200AA_OK iff the current device is sm_90 */

/* CUDA graph capture.  These device entry points may be called on a stream that is capturing a graph (any capture mode),
 * and the graph's replays give their eager results bit for bit: b200aa_clip_stats, b200aa_st_features, b200aa_spectrogram,
 * b200aa_chromagram (and _ragged), b200aa_frame_counts, b200aa_row_counts, b200aa_mid_pool (and _ragged),
 * b200aa_long_term_mean (and _ragged), b200aa_beat_extraction, and their _f64 forms.  A captured launch of a persistent
 * kernel takes its work slot from stream-ordered scratch (an allocation and a free node of the graph) instead of the plan's
 * ring, so no graph shares a slot with another launch or replay.  Every other device entry point, the host-buffer entry
 * points, b200aa_plan_create and b200aa_trees_create return B200AA_ERR_CAPTURE on a capturing stream before any other CUDA
 * call, and so does a float64 call whose plan has not built its float64 tables in an eager call yet.  The entry points
 * without a stream argument can only see the legacy default stream: they refuse when it is capturing, or when a blocking
 * stream captures and any use of it would break that capture.  A plan a graph uses must outlive the graph. */

/* ------------------------------------------------------------------ host tables -------
 * Pure host code, usable without a GPU (the CPU test-suite checks them against the oracle).
 *   which = 0: mel filterbank, dense [40 x K] doubles           (mfcc_filter_banks, ShortTermFeatures.py:191-233)
 *   which = 1: chroma operator, dense [12 x K] doubles           (chroma_features_init + scatter, :257-302)
 *   which = 2: DCT-II ortho rows 0..12, dense [13 x 40] doubles  (scipy dct call at :253)
 * K = window / 2.  Returns B200AA_ERR_CHROMA / B200AA_ERR_MEL_RANGE where the reference raises. */
int b200aa_host_table(int fs, int window, int which, double *h_out);

/* frame / row counts of the three reference entry points */
int64_t b200aa_num_frames(int64_t n_samples, int window, int step);            /* ShortTermFeatures.py:608 */
int64_t b200aa_spectrogram_rows(int64_t n_samples, int window, int step);      /* :413 */
int64_t b200aa_chromagram_rows(int64_t n_samples, int window, int step);       /* :347 */
int64_t b200aa_mid_windows(int64_t n_frames, int step_ratio);                  /* MidTermFeatures.py:116-124 */

/* ------------------------------------------------------------------ plan --------------- */
int  b200aa_plan_create(b200aa_plan **out, int fs, int window, int step);
void b200aa_plan_destroy(b200aa_plan *plan);
/* kernel that feature launches of this plan use: 0 = generic mixed-radix kernel (any window), 1 = register-tiled
 * CTA kernel (windows 320/400/480/600/640/800/882), 2 = warp-autonomous pair kernel (windows 32*R: 320/480/512/640/
 * 800/960/1024), 3 = warp-autonomous per-frame kernel (windows 882/400/600, also their spectrogram / chromagram rows) */
int  b200aa_plan_kernel_kind(const b200aa_plan *plan);
/* restrict the plan to one kernel (testing / A-B runs): -1 = automatic (default), 0..3 as above; a kind that
 * does not exist for the plan's window falls through to the next one */
int  b200aa_plan_prefer_kernel(b200aa_plan *plan, int kind);
/* force the generic kernel (testing): returns the previous setting */
int  b200aa_plan_force_generic(b200aa_plan *plan, int on);

/* frees the device workspaces the host entry points keep between calls (grown to the largest call seen) */
int  b200aa_plan_trim(b200aa_plan *plan);

/* ------------------------------------------------------------------ device entry points */

/* Kernel 0: per-clip statistics -> normalisation records.
 * d_sig: [n_clips] clips, clip b starts at element b*clip_stride; d_len (nullable, int64[n_clips])
 * gives ragged lengths (<= n_samples); d_norm: [n_clips] records.
 * Replaces: `signal / 2**15` + dc_normalize (ShortTermFeatures.py:567-570, :14-19). */
int b200aa_clip_stats(const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                      int64_t clip_stride, const int64_t *d_len,
                      b200aa_clip_norm *d_norm, void *stream);

/* Kernel 1: fused short-term features.  d_out: float32 [n_clips, F, t_stride] with
 * F = 34 (deltas == 0) or 68, frame t of clip b, feature f at d_out[(b*F + f)*t_stride + t];
 * t_stride >= frames of the longest clip.  Columns >= the clip's own frame count are not written.
 * Replaces: the frame loop of ShortTermFeatures.feature_extraction (:608-685). */
int b200aa_st_features(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                       int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                       const b200aa_clip_norm *d_norm, int deltas,
                       float *d_out, int64_t t_stride, void *stream);

/* Spectrogram rows: d_out float32 [n_clips, R, K], R = b200aa_spectrogram_rows(n_samples),
 * trailing rows zero exactly as the reference leaves them (ShortTermFeatures.py:413-422). */
int b200aa_spectrogram(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                       int64_t n_samples, int64_t clip_stride,
                       const b200aa_clip_norm *d_norm, float *d_out, void *stream);

/* Chromagram rows: d_out float32 [n_clips, R, 12], R = b200aa_chromagram_rows(n_samples)
 * (ShortTermFeatures.py:347-359), including the zero last row / clipped last frame cases. */
int b200aa_chromagram(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                      int64_t n_samples, int64_t clip_stride,
                      const b200aa_clip_norm *d_norm, float *d_out, void *stream);

/* Spectrogram / chromagram rows of a ragged batch: clip b is the first d_len[b] samples (int64 [n_clips] on the device,
 * at most n_samples) of its row of d_sig; d_norm from b200aa_clip_stats with the same d_len.  d_out float32
 * [n_clips, R, K] (spectrogram) / [n_clips, R, 12] (chromagram) with R = b200aa_spectrogram_rows(n_samples) /
 * b200aa_chromagram_rows(n_samples), the rows of the widest possible clip.  Clip b's rows below R_b =
 * b200aa_row_counts(d_len)[b] are bit for bit what b200aa_spectrogram / b200aa_chromagram give for the clip alone
 * (zero rows included); rows >= R_b are not written, and a clip the single-clip entry point refuses (R_b = 0) gets
 * nothing written.  NULL pointers, clip_stride < n_samples and a bad dtype are B200AA_ERR_INVALID; R <= 0 is
 * B200AA_ERR_TOO_SHORT; a plan whose chroma table the reference cannot build makes the chromagram entry point return
 * B200AA_ERR_CHROMA for the whole batch.  Nothing synchronises: the counts never leave the device.
 * Replaces: spectrogram() / chromagram() (ShortTermFeatures.py:324-452) of every file of a set of different lengths. */
int b200aa_spectrogram_ragged(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                              int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                              const b200aa_clip_norm *d_norm, float *d_out, void *stream);
int b200aa_chromagram_ragged(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                             int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                             const b200aa_clip_norm *d_norm, float *d_out, void *stream);

/* Per-clip rows of a ragged spectrogram (which = 0) or chromagram (which = 1), computed on the device: d_rows int64
 * [n_clips] = b200aa_spectrogram_rows / b200aa_chromagram_rows(d_len[b]), or 0 for a clip b200aa_spectrogram /
 * b200aa_chromagram refuse (every accepted clip has at least one row).  NULL pointers, n_clips < 0, window < 1,
 * step < 1 and another `which` are B200AA_ERR_INVALID.  Nothing synchronises. */
int b200aa_row_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int which, int64_t *d_rows,
                      void *stream);

/* Kernel 2: mid-term pooling.  d_st float32 [n_clips, F, t_stride] (n_frames valid columns),
 * d_mid float32 [n_clips, 2F, M], M = b200aa_mid_windows(n_frames, step_ratio): rows 0..F-1 means,
 * F..2F-1 population standard deviations of st[f][c : min(c+ratio, T)], c = j*step_ratio.
 * The window is a Python slice, as in the reference: ratio may be 0 or negative (the reference's round() of
 * (mid_window - (short_window - short_step)) / short_step gives that for short mid-term windows).  A negative end
 * counts from the end of the row (ratio -1: window 0 is st[f][0 : T-1]); an empty window gives mean = std = 0
 * (np.nan_to_num of the NaNs of an empty slice).  step_ratio < 1 is B200AA_ERR_INVALID: the reference's window
 * loop never ends there.
 * Replaces: MidTermFeatures.mid_feature_extraction's pooling loops (:110-126). */
int b200aa_mid_pool(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames,
                    int64_t t_stride, int ratio, int step_ratio, float *d_mid, void *stream);

/* Long-term average (SURVEY 8f rank 1): d_out float32 [n_clips, n_rows], the mean of every row of
 * d_mid [n_clips, n_rows, n_windows] over the windows.
 * Replaces: `mid_features.mean(axis=0)` in directory_feature_extraction (MidTermFeatures.py:200-201). */
int b200aa_long_term_mean(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows,
                          float *d_out, void *stream);

/* Per-clip counts of a ragged batch, computed on the device from its lengths: d_len int64 [n_clips] (the lengths given to
 * b200aa_clip_stats / b200aa_st_features); d_frames int64 [n_clips] = b200aa_num_frames(d_len[b], window, step);
 * d_windows (nullable) int64 [n_clips] = b200aa_mid_windows(d_frames[b], step_ratio).  NULL d_len / d_frames,
 * window < 1, step < 1, and step_ratio < 1 with d_windows are B200AA_ERR_INVALID.  Lets a caller that holds the lengths
 * only on the device pass the counts below without a round trip to the host. */
int b200aa_frame_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int step_ratio,
                        int64_t *d_frames, int64_t *d_windows, void *stream);

/* Kernel 2 on a ragged batch: d_st float32 [n_clips, n_feats, t_stride]; d_frames int64 [n_clips]: clip b has
 * T_b = clamp(d_frames[b], 0, t_stride) frames and M_b = b200aa_mid_windows(T_b, step_ratio) windows.  d_mid float32
 * [n_clips, 2 * n_feats, M], M = b200aa_mid_windows(t_stride, step_ratio); columns >= M_b of clip b are not written.
 * Windows, ratio and step_ratio as in b200aa_mid_pool, with T_b for n_frames.  A clip's columns are bit for bit those
 * b200aa_mid_pool gives for it alone with n_frames = T_b: each window's sums run in an order set by the window's bounds
 * only.  NULL pointers, n_feats < 1, step_ratio < 1 and t_stride < 0 are B200AA_ERR_INVALID.
 * Replaces: the pooling loops (MidTermFeatures.py:110-126) of every file of a folder of files of different lengths. */
int b200aa_mid_pool_ragged(const float *d_st, int64_t n_clips, int n_feats, int64_t t_stride,
                           const int64_t *d_frames, int ratio, int step_ratio, float *d_mid, void *stream);

/* Long-term average on a ragged batch: d_mid float32 [n_clips, n_rows, m_stride]; d_windows int64 [n_clips]: clip b
 * averages its first M_b = clamp(d_windows[b], 0, m_stride) columns, NaN for M_b = 0 (0 / 0, as np.mean of an empty
 * axis).  d_out float32 [n_clips, n_rows], bit for bit b200aa_long_term_mean of the clip alone with n_windows = M_b.
 * NULL pointers, n_rows < 1 and m_stride < 0 are B200AA_ERR_INVALID.
 * Replaces: `mid_features.mean(axis=0)` (MidTermFeatures.py:200-201) of every file of a folder. */
int b200aa_long_term_mean_ragged(const float *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                 const int64_t *d_windows, float *d_out, void *stream);

/* Feature vectors for the classifiers that consume the mid-term matrix (SURVEY 8f rank 4): d_out float32
 * [n_clips, n_windows, n_rows], vector j of clip b = (d_mid[b, :, j] - mean) / std -- the transpose the per-window loops
 * build one column at a time.  d_mean / d_std: float32 [n_rows] on the device.
 * Replaces: `feature_vector = (mt_feats[:, col_index] - mean) / std` per window (audioSegmentation.py:581-584,
 * audioTrainTest.py:1091) and per short-term frame (audioSegmentation.py:744-748, with d_mid = the [68 x T] matrix). */
int b200aa_normalize_windows(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows,
                             const float *d_mean, const float *d_std, float *d_out, void *stream);

/* ------------------------------------------------------------------ float64 path (kernel family 12)
 * The float64 counterparts of the entry points above: the same arguments, float64 outputs, and d_sig may also be
 * float64 (B200AA_DTYPE_F64, read unrounded).  Every value is computed in float64 as the float64 oracle computes it
 * (csrc/f64.cuh): the normalisation and rows 0-1 (zcr, energy) bit for bit NumPy, the transform an fp64 mixed-radix
 * FFT, the other rows in the order of the oracle's loop.  Argument checks and refusals are the float32 entry points'. */

/* Normalisation records of the float64 path: d_norm [n_clips] (d_len as in b200aa_clip_stats). */
int b200aa_clip_stats_f64(const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples, int64_t clip_stride,
                          const int64_t *d_len, b200aa_clip_norm_f64 *d_norm, void *stream);
/* d_out float64 [n_clips, F, t_stride] as b200aa_st_features; d_norm from b200aa_clip_stats_f64 with the same d_len. */
int b200aa_st_features_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                           int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm_f64 *d_norm, int deltas,
                           double *d_out, int64_t t_stride, void *stream);
int b200aa_spectrogram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                           int64_t clip_stride, const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream);
int b200aa_spectrogram_ragged_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                  int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                  const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream);
int b200aa_chromagram_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                          int64_t clip_stride, const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream);
int b200aa_chromagram_ragged_f64(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                 int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                 const b200aa_clip_norm_f64 *d_norm, double *d_out, void *stream);
/* Mid-term pooling of float64 rows, bit for bit np.mean / np.std of each window and np.nan_to_num
 * (MidTermFeatures.py:110-126); windows, ratio and step_ratio as in b200aa_mid_pool / b200aa_mid_pool_ragged. */
int b200aa_mid_pool_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                        int ratio, int step_ratio, double *d_mid, void *stream);
int b200aa_mid_pool_ragged_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t t_stride,
                               const int64_t *d_frames, int ratio, int step_ratio, double *d_mid, void *stream);
/* Long-term mean of float64 mid-term rows, bit for bit `mid.T.mean(axis=0)` (MidTermFeatures.py:200-201); windows as in
 * b200aa_long_term_mean / b200aa_long_term_mean_ragged. */
int b200aa_long_term_mean_f64(const double *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, double *d_out,
                              void *stream);
int b200aa_long_term_mean_ragged_f64(const double *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                     const int64_t *d_windows, double *d_out, void *stream);

/* PCM WAV decode (SURVEY 8f rank 2): data-chunk formats of a byte arena, as scipy.io.wavfile.read returns them */
#define B200AA_PCM_U8 0           /* PCM 8-bit, unsigned                                        */
#define B200AA_PCM_S16 1          /* PCM 16-bit                                                 */
#define B200AA_PCM_S24 2          /* PCM 24-bit, packed (scipy: int32, the 3 bytes shifted left by 8) */
#define B200AA_PCM_S32 3          /* PCM 32-bit                                                 */
#define B200AA_PCM_F32 4          /* IEEE float 32                                              */
#define B200AA_PCM_F64 5          /* IEEE float 64                                              */

/* One clip of the arena: n_frames interleaved frames of `channels` (1 or 2) little-endian samples of `format`, starting
 * at byte `offset` (a multiple of 16).  The clip's slot runs from offset to offset + n_frames * block rounded up to a
 * multiple of 16 (block = channels * sample bytes) and is zero past the frames.  24 bytes. */
typedef struct b200aa_pcm_clip {
    int64_t offset;
    int64_t n_frames;
    int32_t format;
    int32_t channels;
} b200aa_pcm_clip;

/* Decode a ragged batch of WAV data chunks: d_out [n_clips, n_out] of out_dtype (B200AA_DTYPE_I16 / _F32), row b at
 * d_out + b * out_stride elements.  out[b, i] for i < n_frames of clip b is the frame converted as
 * _as_clip(stereo_to_mono(wavfile.read(path)[1])) stages it (csrc/pcm.cuh: mono U8 / S16 as int16, every other flavour
 * as float32; NaN stays NaN, its payload may differ), and 0 for n_frames <= i < n_out; every element is written.
 * h_clips is HOST memory and every descriptor is checked before any CUDA call: NULL pointers, n_clips < 0, n_out < 0,
 * out_stride < n_out, an unknown format, channels other than 1 or 2, a negative or misaligned offset, n_frames < 0 or
 * > n_out, a slot past arena_bytes, and out_dtype int16 for anything but mono U8 / S16 are B200AA_ERR_INVALID.  The
 * descriptors are then copied to stream-ordered scratch; nothing synchronises.
 * Replaces: wavfile.read + stereo_to_mono + the float32 cast (audioBasicIO.py:86-110, :156-168) of every file of a
 * folder, on the host. */
int b200aa_decode_pcm(const void *d_arena, int64_t arena_bytes, const b200aa_pcm_clip *h_clips, int64_t n_clips,
                      int out_dtype, void *d_out, int64_t n_out, int64_t out_stride, void *stream);

/* Kernel 4: beat rate of every clip from its short-term rows 0, 1, 3 .. 18 (SURVEY 8f rank 4).  d_st: float32
 * [n_clips, n_feats, t_stride], n_feats >= 19; d_frames (nullable, int64 [n_clips]): frames of each clip, clamped to
 * [0, n_frames]; else n_frames for every clip.  d_out: float64 [n_clips, 2] = (bpm, ratio), bit for bit the host
 * beat_extraction(st[b, :, :T_b] widened to float64, window_size), NaN where it gives NaN (a clip of 0 frames).
 * The histogram has round(2 / window_size) bins (half to even); fewer than 1 is B200AA_ERR_INVALID, as are n_feats < 19,
 * t_stride < n_frames and n_frames >= 2^31 - 1024.  Allocates stream-ordered scratch (at most 256 MiB) on `stream`.
 * Replaces: MidTermFeatures.beat_extraction (:18-84) and utilities.peakdet (:33-103). */
int b200aa_beat_extraction(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                           const int64_t *d_frames, double window_size, double *d_out, void *stream);
/* Kernel 4 on float64 rows (the float64 path's short-term features): the same arguments and result, bit for bit the host
 * beat_extraction(st[b, :, :T_b], window_size). */
int b200aa_beat_extraction_f64(const double *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                               const int64_t *d_frames, double window_size, double *d_out, void *stream);

/* Kernel 5: the library's kNN classifier on a matrix of query vectors (SURVEY 8f rank 4).  Training set on the device:
 * d_feats float64 [n_train, n_feats]; d_slots int32 [n_train], the class a training row votes for (its label when that is
 * an integer in [0, n_classes), else -1: never counted); n_classes = len(np.unique(labels)); k = the model's neighbors.
 * d_query: [n_query] rows of n_feats float32 (B200AA_DTYPE_F32, widened exactly) or float64 (B200AA_DTYPE_F64), row q at
 * element q * q_stride.  d_ids int64 [n_query], d_P float64 [n_query, n_classes]: row q is Knn.classify(query q) bit for
 * bit -- distances summed in sequence in fp64 without FMA as scipy's cdist does, the k smallest (distance, training index)
 * pairs with every NaN after +inf (all n_train of them when k >= n_train), P[c] = count / k, the id the first maximum.
 * The reference's own argsort leaves only an exact tie at the k-th place between different classes open; there the lower
 * training index is taken.  NULL pointers, n_train < 1 (or >= 2^31), n_feats < 1, n_classes < 1, k < 1, n_query < 0,
 * q_stride < n_feats and another dtype are B200AA_ERR_INVALID, checked before any CUDA call; n_query = 0 does nothing.
 * Allocates stream-ordered scratch of one 8-byte key per (query, training row), queries in slices of at most 256 MiB.
 * Replaces: audioTrainTest.Knn.classify (:33-49) per window in classifier_wrapper (:52-93). */
int b200aa_knn_classify(const double *d_feats, const int32_t *d_slots, int64_t n_train, int n_feats, int n_classes,
                        int64_t k, const void *d_query, int dtype, int64_t n_query, int64_t q_stride, int64_t *d_ids,
                        double *d_P, void *stream);

/* Kernel 6: the model selection of audioTrainTest.evaluate_classifier (:576-771) for the library's kNN, every
 * (neighbour count, train / test split) problem of it in one batch.  Device: d_X float64 [n, n_feats] (row i at
 * i * n_feats), d_y int32 [n] each row's class index.  Host: per problem p < n_problems, its training rows
 * h_train_idx[h_train_off[p] .. h_train_off[p + 1]) and test rows h_test_idx[h_test_off[p] .. h_test_off[p + 1]) (int32
 * row indices, in split order; both offset arrays hold n_problems + 1 entries from 0), its k h_k[p] and the class count
 * of its training rows h_classes[p] (len(np.unique(y_train))).  Per problem the training rows are standardised as
 * StandardScaler().fit(X_train).transform does it (scikit-learn 1.9: sequential sums in split order, its constant-column
 * rule), the test rows with the same mean_ / scale_, and each test row is classified as Knn(X_train, y_train, k).classify
 * (kernel 5's contract; a training row votes for its class when that is below h_classes[p]; an exact tie at the k-th
 * place between different classes goes to the lower position in the split).  Writes d_pred int32 [h_test_off[n_problems]],
 * the predicted class of each test row in the same order, and d_counts int64 [n_problems, n_classes, n_classes], per
 * problem the count of test rows of class y_test predicted as y_pred at [y_test, y_pred] (a y outside [0, n_classes) is
 * never counted and never votes).  NULL pointers, n < 1 (or >= 2^31), n_feats < 1, n_classes < 1, n_problems < 0,
 * offsets not from 0, an empty training or test list, an index outside [0, n), k < 1 and h_classes outside
 * [1, n_classes] are B200AA_ERR_INVALID, checked before any CUDA call; n_problems = 0 does nothing.  The index lists
 * are uploaded once; stream-ordered scratch holds the standardised rows and keys of the problems in slices of at most
 * 256 MiB, a problem too large for one slice cut by its test rows.
 * Replaces: the param / experiment loop of evaluate_classifier for classifier_name "knn" without SMOTE. */
int b200aa_knn_cross_validate(const double *d_X, const int32_t *d_y, int64_t n, int n_feats, int n_classes,
                              int64_t n_problems, const int64_t *h_train_off, const int32_t *h_train_idx,
                              const int64_t *h_test_off, const int32_t *h_test_idx, const int64_t *h_k,
                              const int32_t *h_classes, int32_t *d_pred, int64_t *d_counts, void *stream);

/* Kernel 7 (csrc/hmm.cuh): HMM segmentation with the library's diagonal-Gaussian HMMs (audioSegmentation.py:287-344,
 * :471-492).
 *
 * b200aa_hmm_statistics: the means and standard deviations of train_hmm_compute_statistics.  d_mid is a
 * [n_clips, n_feats, m_stride] batch of float32 (B200AA_DTYPE_F32, widened exactly) or float64 (B200AA_DTYPE_F64); clip b
 * contributes its first h_n_windows[b] columns (0 .. m_stride) to one concatenated sequence of windows.  Class c's windows
 * are h_idx[h_class_off[c] .. h_class_off[c + 1]), indices into that sequence in the order NumPy meets them.  Writes d_out
 * [4, n_classes, n_feats] float64: per (class, feature) the sum, the mean (sum / n), the sum of squared deviations and the
 * population std, bit for bit NumPy's mean / std of features[:, idx] (a sequential sum over the windows, pairwise for
 * n_feats == 1).  A class of no windows gives NaN.  NULL pointers, n_clips / n_feats / m_stride / n_classes < 1, a count
 * outside [0, m_stride], offsets not from 0 or decreasing and an index outside [0, sum of the counts) are
 * B200AA_ERR_INVALID, checked before any CUDA call.
 *
 * b200aa_hmm_decode: GaussianHMM(C, "diag").predict of each clip's windows (hmmlearn's Viterbi; ties: the last state is the
 * first maximum, every backtrack step the last maximal predecessor).  d_mid [n_clips, n_feats, m_stride] float32, clip b's
 * first h_n_windows[b] (1 .. m_stride) columns.  The model, on the device, from the host: d_log_start [C] = log pi,
 * d_log_trans [C, C] = log A (-inf for a zero probability), d_means [C, n_feats], d_vars [C, n_feats] the diagonal
 * covariances (> 0), d_const [C] = n_feats log 2pi + sum_f log var.  Writes d_ids int32 [n_clips, m_stride], each clip's
 * states and zeros past its count, and d_bad int32 [n_clips]: 1 for a clip with a non-finite feature, whose ids are not
 * written.  C = n_states in [1, 2048].  NULL pointers, counts below 1 and a count above m_stride are B200AA_ERR_INVALID,
 * checked before any CUDA call.  Stream-ordered scratch holds the emissions and backpointers of the clips in slices of at
 * most 256 MiB (a clip larger than that on its own takes a slice of its own). */
int b200aa_hmm_statistics(const void *d_mid, int dtype, int64_t n_clips, int n_feats, int64_t m_stride,
                          const int64_t *h_n_windows, int n_classes, const int64_t *h_class_off, const int64_t *h_idx,
                          double *d_out, void *stream);
int b200aa_hmm_decode(const float *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, const int64_t *h_n_windows,
                      int n_states, const double *d_log_start, const double *d_log_trans, const double *d_means,
                      const double *d_vars, const double *d_const, int32_t *d_ids, int32_t *d_bad, void *stream);

/* b200aa_hmm_decode_f64: b200aa_hmm_decode of float64 windows, the same model arguments, outputs and checks.  Clip b is
 * d_mid + b * n_feats * m_stride: with window_major = 0 a [n_feats, m_stride] matrix (the layout b200aa_hmm_decode reads;
 * predict(features.T) sums a window's density terms in sequence), with window_major = 1 a C-contiguous [m_stride, n_feats]
 * matrix of one window per row (predict(X) of a C-contiguous X sums them pairwise, NumPy's order for a contiguous row).
 * window_major other than 0 / 1 is B200AA_ERR_INVALID. */
int b200aa_hmm_decode_f64(const double *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, int window_major,
                          const int64_t *h_n_windows, int n_states, const double *d_log_start, const double *d_log_trans,
                          const double *d_means, const double *d_vars, const double *d_const, int32_t *d_ids, int32_t *d_bad,
                          void *stream);

/* Kernel 9 (csrc/cluster.cuh): the cluster distance means of speaker_diarization's silhouette (audioSegmentation.py:943-985)
 * for one clustering of the n rows of d_X (float64, row r at d_X + r * x_stride, n_feats columns), h_labels [n] on the host,
 * each in [0, n_clusters).  For every cluster c with h_want[c] != 0 (h_want NULL: every cluster), X_c its rows in ascending
 * order, writes d_A[c] = np.mean(pdist(X_c.T)) and d_B[c * K + c2] = np.mean(cdist(X_c, X_c2)) for c2 != c, float64, bit
 * for bit scipy's sequential euclidean chain and NumPy's pairwise sum of the condensed vector / the row-major block, then
 * one division by the count.  A mean of no terms (n_feats < 2 for A, an empty X_c2 for B), a diagonal entry and the rows
 * of clusters not wanted are NaN.  NULL pointers (h_want aside), n < 1, n_feats outside [1, 4096], x_stride < n_feats,
 * n_clusters outside [1, B200AA_CLUSTER_MAX] and a label outside [0, n_clusters) are B200AA_ERR_INVALID, before any CUDA
 * call.  Stream-ordered scratch: the gathered rows (n x n_feats doubles) and the distances of one pass (at most 128 MiB,
 * or one segment of a mean's pairwise tree when that is larger). */
#define B200AA_CLUSTER_MAX 1024
int b200aa_cluster_distance_means(const double *d_X, int64_t n, int n_feats, int64_t x_stride, const int32_t *h_labels,
                                  int n_clusters, const unsigned char *h_want, double *d_A, double *d_B, void *stream);

/* Kernel 10 (csrc/thumb.cuh): music_thumbnailing's self-similarity matrix, diagonal filter, masked argmax and walk
 * (audioSegmentation.py:40-55, :1093-1180) for a ragged batch of n_tracks standardised tracks.  Track b is h_frames[b]
 * consecutive rows of d_X (float64, row r at d_X + r * x_stride, n_feats columns, one frame per row), after the rows of the
 * tracks before it.  Bit for bit scipy and NumPy:
 *   S = 1 - squareform(pdist(X_b, 'cosine'))       scipy's two-accumulator dot product, no FMA; 1.0 on the diagonal
 *   C = convolve2d(S, eye(filter_len), 'valid')    R_b = T_b - filter_len + 1; NaN when any entry of the box is NaN
 *   entries with |i - j| < diag_gap, i > j, or a row or column outside [h_limits[2b], h_limits[2b + 1]) set to np.min(C)
 *   the first maximum in row-major order (the first NaN when there is one), then the reference's walk.
 * Two modes.  d_sim non-NULL (d_out and d_idx NULL): only S, track b's [T_b, T_b] at d_sim + sum_{c<b} T_c^2.  Otherwise
 * d_out receives the masked C, track b's [R_b, R_b] at d_out + sum_{c<b} R_c^2, and d_idx[4b ..] (i1, i2, j1, j2), frame
 * indices (the reference returns short_step times these).  NULL pointers, n_feats < 1, x_stride < n_feats, n_tracks < 1,
 * T_b < 1 or above 2^28, and for the filter filter_len < 1, T_b < filter_len or limits outside [0, R_b] are
 * B200AA_ERR_INVALID, before any CUDA call.  Stream-ordered scratch: the row norms, and S plus T_b x R_b bytes of NaN
 * windows for a slice of tracks of at most 256 MiB (a larger track is a slice of its own). */
int b200aa_music_thumbnail(const double *d_X, int n_feats, int64_t x_stride, const int64_t *h_frames, int64_t n_tracks,
                           int filter_len, double diag_gap, const int64_t *h_limits, double *d_sim, double *d_out,
                           int64_t *d_idx, void *stream);

/* Kernel 11 (csrc/front.cuh): the host steps of speaker_diarization and music_thumbnailing between the features and
 * kernels 9 and 10, bit for bit scikit-learn 1.9, scipy and NumPy.
 *
 * b200aa_standard_scale: StandardScaler().fit_transform of each of n_mats matrices.  Matrix b has h_rows[b] rows and n_feats
 * columns, entry (i, j) at d_X + b * mat_stride + i * row_stride + j * col_stride, float32 (widened) or float64
 * (B200AA_DTYPE_F32 / F64).  Its columns are summed as np.sum / np.nansum over axis 0 sums them: pairwise down each column
 * when row_stride < col_stride or n_feats == 1, else row by row.  NaN is left out of the sums and the counts and passes
 * through.  Writes entry (i, j) of the result at d_out + h_out_off[b] + i * out_row_stride + j * out_col_stride, and
 * d_mean / d_scale [n_mats, n_feats] (scikit-learn's mean_ and scale_), and d_bad int32 [n_mats]: 1 for a matrix holding
 * +-inf, which scikit-learn refuses and whose outputs are meaningless.  NULL pointers, n_mats < 1, n_feats < 1, a row count
 * below 1, a negative offset or mat_stride, strides below 1 and an unknown dtype are B200AA_ERR_INVALID, before any CUDA
 * call.  Stream-ordered scratch: the row counts and offsets.
 *
 * b200aa_outlier_columns: the feature-outlier rule of speaker_diarization (audioSegmentation.py:861-865) for the
 * normalised [n_rows, n_feats] matrix X, column u at d_X + u * col_stride (its n_rows values contiguous): d_dist_all
 * [n_feats] = np.sum(squareform(pdist(X.T)), axis=0), *d_mean = np.mean(dist_all), d_keep [n_feats] = dist_all < 1.1 *
 * mean (1 / 0).  NULL pointers, n_rows < 1, n_feats outside [1, 4096] and col_stride outside [n_rows, INT_MAX] are
 * B200AA_ERR_INVALID, before any CUDA call.  Stream-ordered scratch: the n_feats^2 distances.
 *
 * b200aa_pool_frames: the LDA branch's pooling (audioSegmentation.py:884-906) of n_clips [n_feats, T_b] matrices, entry
 * (f, i) of clip b at d_st + b * clip_stride + f * row_stride + i, float32 (widened) or float64, T_b = h_frames[b]:
 * d_out [n_clips, 2 n_feats, out_stride] float64, row f of clip b at frame i the np.mean and row n_feats + f the np.std of
 * frames [i, min(i + ratio, T_b)) of row f; entries past T_b are not written.  NULL pointers, n_clips < 1, n_feats < 1,
 * ratio < 1, negative strides, a frame count outside [1, out_stride] and an unknown dtype are B200AA_ERR_INVALID, before
 * any CUDA call. */
int b200aa_standard_scale(const void *d_X, int dtype, int64_t n_mats, int n_feats, const int64_t *h_rows, int64_t mat_stride,
                          int64_t row_stride, int64_t col_stride, double *d_out, const int64_t *h_out_off,
                          int64_t out_row_stride, int64_t out_col_stride, double *d_mean, double *d_scale, int32_t *d_bad,
                          void *stream);
int b200aa_outlier_columns(const double *d_X, int64_t n_rows, int n_feats, int64_t col_stride, double *d_dist_all,
                           double *d_mean, unsigned char *d_keep, void *stream);
int b200aa_pool_frames(const void *d_st, int dtype, int64_t n_clips, int n_feats, int64_t clip_stride, int64_t row_stride,
                       const int64_t *h_frames, int64_t ratio, double *d_out, int64_t out_stride, void *stream);

/* Kernel 8 (csrc/trees.cuh): the tree classifiers of extract_features_and_train (audioTrainTest.py:52-93), bit for bit
 * scikit-learn 1.9's predict / predict_proba of RandomForestClassifier, ExtraTreesClassifier (mode 0, forest mean) and
 * GradientBoostingClassifier (mode 1, boosting sum).
 *
 * b200aa_trees_create: validates an ensemble on the host and uploads it once to the current device.  h_nodes [n_nodes]:
 * tree t is nodes [h_roots[t], h_roots[t + 1]) (the last up to n_nodes), h_roots[0] = 0.  An internal node has left / right
 * indices into h_nodes, both after the node and inside its tree, a feature in [0, n_feats) (bit 31 set: a NaN goes left)
 * and a float32 threshold, scikit-learn's rounded toward -inf; a leaf has left < 0 and right = its row of h_values, in
 * [0, n_leaves).  Mode 0: h_values [n_leaves, n_classes], every tree votes for every class, P = the per-class sum over the
 * trees in order divided by n_trees, h_init ignored (the sums start at 0).  Mode 1: h_values [n_leaves], the learning rate
 * already applied; tree t adds to class t mod K (K = n_classes) starting from h_init [K].  allow_nan: NaN queries are
 * walked (else the row is flagged).  Anything else is B200AA_ERR_INVALID, before any CUDA call; a row of more shared
 * memory than kernel 8 takes is B200AA_ERR_UNSUPPORTED.  Create returns once the model is on the device, so any stream
 * may use it at once; the model is read-only: any number of streams and threads may classify with it at once.
 * b200aa_trees_destroy waits for the device's queued work before it frees the model.
 *
 * b200aa_trees_classify: d_query [n_query, q_stride], float32 or float64 (B200AA_DTYPE_F32 / F64), n_feats columns
 * read per row, cast to float32 as scikit-learn casts.  Writes d_ids int64 [n_query] (class index: the first maximum
 * of the scores, or raw >= 0 for K = 1), d_scores float64 [n_query, n_classes] (P in mode 0, the raw scores in mode 1) and
 * d_bad int32 [n_query]: 1 for a row scikit-learn refuses (a value that is or becomes +-inf as float32, or NaN unless
 * allowed), whose other outputs are meaningless.  NULL pointers, n_query < 0, n_feats other than the model's, q_stride <
 * n_feats, an unknown dtype are B200AA_ERR_INVALID before any CUDA call; a model of another device too.  n_query = 0 does
 * nothing.  No scratch: every row's work stays in its warp.
 *
 * Replaces: classifier.predict / predict_proba in classifier_wrapper for the three tree model types. */
typedef struct b200aa_tree_node {
    int32_t left, right, feature;
    float threshold;
} b200aa_tree_node;
typedef struct b200aa_trees b200aa_trees;
int b200aa_trees_create(b200aa_trees **out, const b200aa_tree_node *h_nodes, int64_t n_nodes, const int32_t *h_roots,
                        int n_trees, const double *h_values, int64_t n_leaves, int n_classes, int n_feats, int mode,
                        const double *h_init, int allow_nan);
int b200aa_trees_classify(const b200aa_trees *model, const void *d_query, int dtype, int64_t n_query, int n_feats,
                          int64_t q_stride, int64_t *d_ids, double *d_scores, int32_t *d_bad, void *stream);
int b200aa_trees_destroy(b200aa_trees *model);

/* Kernel 13 (csrc/forest.cuh): training of the forests of extract_features_and_train / evaluate_classifier
 * (audioTrainTest.py:52-93), bit for bit scikit-learn 1.9's RandomForestClassifier(n_estimators=T).fit (kind 0, best
 * splitter) and ExtraTreesClassifier(n_estimators=T).fit (kind 1, random splitter) with every other argument at its
 * default: gini, max_features = max(1, int(sqrt(n_feats))), min_samples_split 2, min_samples_leaf 1, no depth limit.
 *
 * b200aa_forest_fit: d_X [n, row_stride] float32 or float64 on the current device (n_feats columns read, cast to float32
 * with round to nearest as fit casts; no NaN and nothing that is or becomes +-inf: the caller refuses those), h_y int32
 * [n] class indices in [0, n_classes), h_weights int32 [n_trees, n] every tree's sample weights (np.bincount of its
 * bootstrap indices) or NULL for weight 1 everywhere, h_seeds uint32 [n_trees] every tree's splitter rand_r_state.
 * Writes the trees one after another to h_nodes / h_values (node_capacity nodes; 2 n - 1 per tree always suffice):
 * tree t has h_node_count[t] nodes in Tree.__getstate__'s order and fields (left / right -1 and feature -2, threshold
 * -2.0 at a leaf) and values [node, n_classes] (class fractions), and h_max_depth[t].  NULL pointers, n < 1 or n > 2^29,
 * n_feats < 1, row_stride < n_feats, n_classes < 1, n_trees < 1, an unknown kind or dtype, max_features outside [1,
 * n_feats], a class index out of range, a negative weight or one above 2^29, and a forest larger than node_capacity are
 * B200AA_ERR_INVALID (all but the last before any CUDA call); more than 512 features or 32 classes is
 * B200AA_ERR_UNSUPPORTED.  Not restated: for kind 1, when a node's minimum of the drawn feature is a zero present with
 * both signs and our_rand_r returns exactly RAND_R_MAX, the stored threshold's zero sign may differ from scikit-learn's
 * (the partition is the same).  One CTA builds one tree; trees run in slices whose stream-ordered scratch stays under 256 MB.
 * The call returns once the nodes are on the host; it refuses a capturing stream (B200AA_ERR_CAPTURE).
 *
 * Replaces: RandomForestClassifier / ExtraTreesClassifier .fit in train_random_forest / train_extra_trees. */
typedef struct b200aa_forest_node {
    int32_t left, right, feature, n_node_samples;
    double threshold, impurity, weighted_n_node_samples;
    int32_t missing_go_to_left, pad;
} b200aa_forest_node;
int b200aa_forest_fit(const void *d_X, int dtype, int64_t n, int n_feats, int64_t row_stride, const int32_t *h_y,
                      int n_classes, int kind, int n_trees, int max_features, const int32_t *h_weights,
                      const uint32_t *h_seeds, b200aa_forest_node *h_nodes, double *h_values, int64_t node_capacity,
                      int64_t *h_node_count, int32_t *h_max_depth, void *stream);

/* b200aa_forest_cross_validate: the model selection of evaluate_classifier (audioTrainTest.py:576-771) for
 * "randomforest" (kind 0) and "extratrees" (kind 1), every (parameter, experiment) problem in one call.  d_X float64
 * [n, n_feats] C-contiguous on the current device, h_y int32 [n] class indices in [0, n_classes).  Problem p trains on
 * rows h_train_idx [h_train_off[p], h_train_off[p + 1]) and tests on h_test_idx [h_test_off[p], h_test_off[p + 1]), in
 * split order (h_train_off[0] = h_test_off[0] = 0).  Per problem, on the device: StandardScaler().fit on the training
 * rows and transform of both (kernel 6's knn::scaler_fit), the forest of h_n_trees[p] trees built by kernel 13 on the
 * training rows cast to float32 with labels the indices into the training rows' sorted classes, and every test row
 * classified as the forest's predict (tree sums in tree order over T, first maximum).  Problem p's trees take
 * h_seeds [sum of the earlier h_n_trees, + h_n_trees[p]) and, for kind 0, h_weights int32 [h_n_trees[p], n_train(p)]
 * (problems one after another; NULL for kind 1, required for kind 0).  Writes d_pred int32 [h_test_off[P]] (each test
 * row's class index) and d_counts int64 [P, n_classes, n_classes] = counts[p, y_test, y_pred], the format of
 * b200aa_knn_cross_validate.  The forests never leave the device.  Argument checks as b200aa_forest_fit's, plus an empty
 * training set, an index outside [0, n) and h_n_trees < 1 are B200AA_ERR_INVALID before any CUDA call.  The call is
 * stream-ordered and returns without waiting for the stream; it refuses a capturing stream. */
int b200aa_forest_cross_validate(const double *d_X, int64_t n, int n_feats, const int32_t *h_y, int n_classes, int kind,
                                 int64_t n_problems, const int64_t *h_train_off, const int32_t *h_train_idx,
                                 const int64_t *h_test_off, const int32_t *h_test_idx, const int32_t *h_n_trees,
                                 const int32_t *h_weights, const uint32_t *h_seeds, int32_t *d_pred, int64_t *d_counts,
                                 void *stream);

/* Kernel 13, regression (csrc/forest.cuh build_regression_tree): scikit-learn 1.9's RandomForestRegressor(n_estimators=T)
 * .fit with the library's arguments (squared_error, max_features=1.0, bootstrap, no depth limit), tree for tree in bits.
 *
 * b200aa_forest_regressor_fit: as b200aa_forest_fit, with h_y float64 [n] finite targets, h_weights int32 [n_trees, n]
 * required (the bootstrap counts), no classes, kind or max_features, and one float64 value per node in h_values
 * [node_capacity].  A non-finite target is B200AA_ERR_INVALID; more than 512 features, or a problem whose single tree's
 * scratch (its sort keys alone take 8 n_feats pow2(n) bytes: at 136 features, n above 131 072) does not fit the 256 MB
 * scratch bound, B200AA_ERR_UNSUPPORTED; all before any CUDA call.  Returns after the stream drained; it refuses a
 * capturing stream.
 * Replaces: RandomForestRegressor.fit in train_random_forest_regression. */
int b200aa_forest_regressor_fit(const void *d_X, int dtype, int64_t n, int n_feats, int64_t row_stride, const double *h_y,
                                int n_trees, const int32_t *h_weights, const uint32_t *h_seeds, b200aa_forest_node *h_nodes,
                                double *h_values, int64_t node_capacity, int64_t *h_node_count, int32_t *h_max_depth,
                                void *stream);

/* b200aa_forest_regression_cross_validate: the "randomforest" model selection of evaluate_regression, every (parameter,
 * experiment) problem in one call.  d_X float64 [n, n_feats] C-contiguous on the current device, h_y float64 [n] finite.
 * The whole matrix is standardised once (kernel 11's scaler: StandardScaler().fit_transform) and cast to float32.
 * Problem p trains on rows h_train_idx [h_train_off[p], h_train_off[p + 1]) and predicts them and its test rows
 * h_test_idx [h_test_off[p], h_test_off[p + 1]) with its forest of h_n_trees[p] trees (seeds h_seeds and weights
 * h_weights int32 [h_n_trees[p], n_train(p)], problems one after another).  The trees of many problems are built in one
 * launch.  Writes float64 predictions (ForestRegressor.predict: tree values added in tree order, then / T) to d_pred_test
 * [h_test_off[P]] and d_pred_train [h_train_off[P]], in split order.  Argument checks as b200aa_forest_regressor_fit's,
 * plus an empty training set, an index outside [0, n) and h_n_trees < 1 are B200AA_ERR_INVALID before any CUDA call
 * (the scratch bound applies to the largest training set together with the call's fixed arrays).  It refuses a
 * capturing stream and waits for its stream between launches.
 * Replaces: the "randomforest" loop of evaluate_regression (train_random_forest_regression and regression_wrapper per
 * problem). */
int b200aa_forest_regression_cross_validate(const double *d_X, int64_t n, int n_feats, const double *h_y, int64_t n_problems,
                                            const int64_t *h_train_off, const int32_t *h_train_idx, const int64_t *h_test_off,
                                            const int32_t *h_test_idx, const int32_t *h_n_trees, const int32_t *h_weights,
                                            const uint32_t *h_seeds, double *d_pred_test, double *d_pred_train, void *stream);

/* Kernel 13, gradient boosting (csrc/forest.cuh boost_leaves): the device side of scikit-learn 1.9's
 * GradientBoostingClassifier(n_estimators=T).fit with the library's arguments (log_loss, learning_rate 0.1, max_depth 3,
 * subsample 1.0), one stage per call.  The caller computes each stage's negative gradient with scikit-learn's own loss
 * (the only step that needs exp / log) and draws every tree's splitter seed; the device builds the stage's trees in bits
 * and does the ordered float64 rest.
 *
 * b200aa_boosting_stage: one stage of many problems.  d_X float32 [n_rows, n_feats] C-contiguous on the current device.
 * Problem p trains on rows h_train_rows [h_train_off[p], h_train_off[p + 1]) (h_train_off[0] = 0) and, when h_test_off /
 * h_test_rows are given (both or neither), also updates its test rows h_test_rows [h_test_off[p], h_test_off[p + 1]).
 * h_n_trees[p] = K, the trees per stage (1: binomial loss, else the multinomial loss over K classes, 3 <= K <= 32), and
 * h_active[p] (0 / 1) whether p fits a tree in this stage.  Device blocks, problems one after another: d_y int32
 * [h_train_off[P]] each training row's class index (0 / 1 for K = 1, else in [0, K)), d_neg_grad float64 and d_raw_train
 * float64 (updated) [n_train(p), K] per problem, d_raw_test float64 (updated) [n_test(p), K] per problem.  h_seeds uint32:
 * the splitter rand_r_state of every tree of the stage, active problems in order, k inner.  Per tree k of an active problem,
 * on its training rows: a DecisionTreeRegressor (squared_error, max_depth 3, every feature, unit weights) on column k of
 * the negative gradient, node for node as build_regression_tree builds it; every leaf's value replaced by
 * _update_terminal_regions' Newton step over the leaf's rows in ascending row order (NumPy pairwise sums, the (K - 1) / K
 * factor for the multinomial loss, 0.0 below |denominator| 1e-150); raw[:, k] += learning_rate * value[leaf] for the
 * training rows and, walking the tree, the test rows.  With h_nodes (and h_values, h_node_count, h_max_depth; all or
 * none) the stage's trees are written as b200aa_forest_fit writes them (one float64 value per node) and the call returns
 * after the stream drained; without, the trees stay on the device and the call is stream-ordered.  NULL pointers,
 * n_rows < 1 or > 2^29, n_feats < 1, n_problems < 1, a non-finite learning_rate, an empty training set, a row outside [0,
 * n_rows), a K outside {1} and [3, 32], an active flag other than 0 / 1, test rows without d_raw_test, and a negative
 * node_capacity are B200AA_ERR_INVALID before any CUDA call, trees beyond node_capacity after; more than 512 features, or
 * a tree whose scratch does not fit the 256 MB scratch bound (its sort keys take 8 n_feats pow2(n_train) bytes),
 * B200AA_ERR_UNSUPPORTED before any CUDA call.  It refuses a capturing stream.
 * Replaces: _fit_stage of GradientBoostingClassifier.fit in train_gradient_boosting, and predict_stages on the test rows
 * of evaluate_classifier's "gradientboosting" branch. */
int b200aa_boosting_stage(const float *d_X, int64_t n_rows, int n_feats, int64_t n_problems, const int64_t *h_train_off,
                          const int32_t *h_train_rows, const int64_t *h_test_off, const int32_t *h_test_rows,
                          const int32_t *h_n_trees, const int32_t *h_active, const int32_t *d_y, const double *d_neg_grad,
                          double *d_raw_train, double *d_raw_test, const uint32_t *h_seeds, double learning_rate,
                          b200aa_forest_node *h_nodes, double *h_values, int64_t node_capacity, int64_t *h_node_count,
                          int32_t *h_max_depth, void *stream);

/* b200aa_boosting_scale: evaluate_classifier's per-split scaling for the boosting model selection.  d_X float64 [n,
 * n_feats] C-contiguous on the current device; per problem p, StandardScaler().fit on rows h_train_idx [h_train_off[p],
 * h_train_off[p + 1]) in split order (kernel 6's knn::scaler_fit) and transform of them and of its test rows h_test_idx
 * [h_test_off[p], h_test_off[p + 1]), cast to float32 as fit and predict cast them.  Writes d_Xs float32 [h_train_off[P] +
 * h_test_off[P], n_feats]: problem p's training rows at row h_train_off[p], its test rows at row h_train_off[P] +
 * h_test_off[p].  NULL pointers, n < 1 or n > 2^29, n_feats < 1, n_problems < 1, an empty training set and an index
 * outside [0, n) are B200AA_ERR_INVALID before any CUDA call.  Stream-ordered; it refuses a capturing stream. */
int b200aa_boosting_scale(const double *d_X, int64_t n, int n_feats, int64_t n_problems, const int64_t *h_train_off,
                          const int32_t *h_train_idx, const int64_t *h_test_off, const int32_t *h_test_idx, float *d_Xs,
                          void *stream);

/* b200aa_boosting_count: the confusion counts of the boosting model selection from the test rows' final raw scores
 * d_raw_test (float64 [n_test(p), K] per problem, problems one after another, K = h_n_trees[p]).  Each row's predicted
 * class is predict's: raw >= 0 for K = 1, else the first maximum, mapped through h_classes int32 [P, 32] (problem p's
 * present classes in sorted order, as label indices in [0, n_classes)).  Writes d_pred int32 [h_test_off[P]] and d_counts
 * int64 [P, n_classes, n_classes] = counts[p, y_test, y_pred] with h_y_test int32 [h_test_off[P]], the format of
 * b200aa_knn_cross_validate.  NULL pointers, n_problems < 1, n_classes outside [2, 32], a bad K, offset or label are
 * B200AA_ERR_INVALID before any CUDA call.  Stream-ordered; it refuses a capturing stream. */
int b200aa_boosting_count(const double *d_raw_test, int64_t n_problems, const int64_t *h_test_off, const int32_t *h_n_trees,
                          const int32_t *h_classes, const int32_t *h_y_test, int n_classes, int32_t *d_pred,
                          int64_t *d_counts, void *stream);

/* ------------------------------------------------------------------ host entry points --
 * Same operations on HOST buffers: pinned or pageable input is copied to the device, the
 * kernels run, the result is copied back and the call returns after the stream drained.
 * These are what a ctypes / cffi binding of the reference would call (INTEGRATION.md). */
int b200aa_st_features_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_clips,
                            int64_t n_samples, int deltas, float *h_out /* [n_clips, F, T] */);
int b200aa_spectrogram_host(const b200aa_plan *plan, const void *h_sig, int dtype,
                            int64_t n_samples, float *h_out /* [R, K] */);
int b200aa_chromagram_host(const b200aa_plan *plan, const void *h_sig, int dtype,
                           int64_t n_samples, float *h_out /* [R, 12] */);
int b200aa_mid_features_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_samples,
                             int ratio, int step_ratio,
                             float *h_mid /* [136, M] */, float *h_st /* [68, T], nullable */);

/* Pinned (page-locked) host buffers for the host entry points: with them the chunked pipeline inside
 * b200aa_st_features_host overlaps the PCIe copies of neighbouring chunks with the kernels.  Pages are placed by
 * the calling thread's NUMA policy -- bind the thread to the GPU's node first (pyaudioanalysis_b200/numa.py).
 * Replaces nothing in the reference (its arrays are pageable NumPy buffers, audioBasicIO.py:86-110); SURVEY 8f rank 2. */
int b200aa_host_alloc(void **h_out, size_t bytes);
int b200aa_host_free(void *h_ptr);

/* Peer-mapped gather target (SURVEY 8e, BASELINE configs[4]): the root rank creates one device buffer for the
 * features of ALL clips and exports a 64-byte handle; every other rank of the box opens it (CUDA IPC, NVLink peer
 * mapping).  A rank then either pushes its finished block with b200aa_peer_copy (copy engines, asynchronous on a
 * stream of its own so the transfer rides under the next batch's kernels; no collective kernel, no SM on either
 * side) or passes `peer_ptr + its slice offset` straight as d_out of b200aa_st_features (the tile stores land in
 * the root's HBM: free at 2 GPUs, but 32-byte remote stores from 7 GPUs into one collapse to ~220 GB/s at 8).
 * Handles travel between the processes by any byte channel (the Python host side uses torch.distributed). */
#define B200AA_IPC_HANDLE_BYTES 64
int b200aa_peer_buffer_create(size_t bytes, void **d_out, unsigned char *handle_out /* [64] */);
int b200aa_peer_buffer_open(const unsigned char *handle /* [64] */, void **d_out);
int b200aa_peer_copy(void *d_dst /* peer-mapped or local */, const void *d_src, size_t bytes, void *stream);
int b200aa_peer_buffer_close(void *d_ptr, int owner /* 1: the creating rank (frees), 0: a mapping rank (unmaps) */);

/* debugging: when set (device pointer, float32 [n_clips, t_stride, K]) the pair kernel also dumps its |X| rows */
int b200aa_debug_set_dump(float *d_rows);

/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t b200aa_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200AA_H_ */
