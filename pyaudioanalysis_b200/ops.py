"""The batched API as PyTorch operators: ``torch.ops.b200aa.*``.

Each operator is functional (it returns new tensors and writes none of its inputs) and calls the ``batch`` function of the
same name, so its results are that function's, bit for bit.  ``torch.compile`` traces them without a graph break, and
each has a fake implementation that gives its output shapes from the clip length and the window arguments alone, with
integer arithmetic that also works on symbolic sizes.  A shape the eager call refuses raises in the fake implementation
too.  The operators are not differentiable.

Inside a CUDA graph capture the library captures the feature path and refuses everything else (include/b200aa.h); plans
come from the cache only (``_lib.get_plan``), so make one eager call of each configuration before capturing it.
"""
from typing import Optional, Tuple

import torch

from . import _lib, batch

_F32 = torch.float32


# ---- the counts of csrc/rows.cuh in Python: b200aa_num_frames, b200aa_spectrogram_rows, b200aa_chromagram_rows and
# b200aa_mid_windows, and whether the equal-length entry points refuse the clip

def _tdiv(a, b):
    """a / b truncated toward zero for b > 0: C's division, and Python's int() of the reference's float quotient."""
    return a // b if a >= 0 else -((-a) // b)


def _range_len(a, b, s):
    """len(range(a, b, s)) for s > 0."""
    return (b - a + s - 1) // s if b > a else 0


def num_frames(n, w, s):
    """Frames of feature_extraction's loop over n samples."""
    return 0 if w < 1 or s < 1 or n < w else (n - w) // s + 1


def spectrogram_rows(n, w, s):
    """(rows of spectrogram's output, True when the equal-length and ragged calls refuse n samples)."""
    if w < 1 or s < 1:
        return 0, True
    R = _tdiv(n - w, s) + 1
    return R, R <= 0 or n == 0


def chromagram_rows(n, w, s):
    """(rows of chromagram's output, True when the equal-length call refuses n samples): no rows, fewer than w + s samples,
    or a clipped last frame shorter than w / 2 samples, where the reference's chroma scatter raises."""
    if w < 1 or s < 1:
        return 0, True
    R = _tdiv(n - s - w, s) + 1
    if R <= 0 or n - s - w < 0:
        return R, True
    n_it = min(R, _range_len(w, n - s, s))
    n_full = min(n_it, (n - 2 * w) // s + 1) if n >= 2 * w else 0
    return R, n_it > n_full and n - (w + (n_it - 1) * s) < w // 2


def mid_windows(n_frames, step_ratio):
    """Mid-term windows of n_frames frames."""
    return 0 if step_ratio < 1 or n_frames <= 0 else (n_frames + step_ratio - 1) // step_ratio


# ---- helpers of the fake implementations

def _refuse(status):
    _lib.check(status)


def _clip_shape(signals):
    """(B, N) of a [B, N] or [N] clip tensor."""
    if signals.dim() == 1:
        return 1, signals.shape[0]
    if signals.dim() != 2:
        raise ValueError("signals must be [B, N] with contiguous samples")
    return signals.shape[0], signals.shape[1]


def _check_dtype(dtype):
    if dtype not in (torch.float32, torch.float64):
        raise TypeError("dtype must be torch.float32 or torch.float64, got %s" % (dtype,))


def _plan_args(window, step):
    w, s = int(window), int(step)
    if w < 2 or s < 1:
        _refuse(_lib.ERR_INVALID)           # b200aa_plan_create
    return w, s


def _frames_or_refuse(N, window, step):
    w, s = _plan_args(window, step)
    T = num_frames(N, w, s)
    if T <= 0:
        _refuse(_lib.ERR_TOO_SHORT)
    return T


def _rows_arg(st, min_feats=1):
    if st.dim() != 3 or st.dtype not in (torch.float32, torch.float64) or st.shape[1] < min_feats:
        raise ValueError("rows must be float32 or float64 [B, F >= %d, T]" % min_feats)
    return st.shape


def _c(t):
    return None if t is None else t.contiguous()


# ---- operators

@torch.library.custom_op("b200aa::clip_stats", mutates_args=(), device_types="cuda")
def clip_stats(signals: torch.Tensor, lengths: Optional[torch.Tensor] = None, dtype: torch.dtype = _F32) -> torch.Tensor:
    """Per-clip normalisation records: uint8 [B, 32] of ``batch.clip_stats`` (float32 path), or [B, 16] of
    ``batch.clip_stats_f64`` (``dtype=torch.float64``)."""
    _check_dtype(dtype)
    if dtype == torch.float64:
        return batch.clip_stats_f64(signals.contiguous(), _c(lengths))
    return batch.clip_stats(signals.contiguous(), _c(lengths))


@clip_stats.register_fake
def _(signals, lengths=None, dtype=_F32):
    _check_dtype(dtype)
    B, _ = _clip_shape(signals)
    nb = batch.NORM_F64_BYTES if dtype == torch.float64 else batch.NORM_BYTES
    return signals.new_empty((B, nb), dtype=torch.uint8)


@torch.library.custom_op("b200aa::feature_extraction", mutates_args=(), device_types="cuda")
def feature_extraction(signals: torch.Tensor, sampling_rate: float, window: float, step: float, deltas: bool = True,
                       lengths: Optional[torch.Tensor] = None, dtype: torch.dtype = _F32) -> torch.Tensor:
    """Short-term features [B, 68 | 34, T] of ``batch.feature_extraction_batch``."""
    return batch.feature_extraction_batch(signals.contiguous(), sampling_rate, window, step, deltas=deltas,
                                          lengths=_c(lengths), dtype=dtype)


@feature_extraction.register_fake
def _(signals, sampling_rate, window, step, deltas=True, lengths=None, dtype=_F32):
    _check_dtype(dtype)
    B, N = _clip_shape(signals)
    T = _frames_or_refuse(N, window, step)
    return signals.new_empty((B, 68 if deltas else 34, T), dtype=dtype)


@torch.library.custom_op("b200aa::spectrogram", mutates_args=(), device_types="cuda")
def spectrogram(signals: torch.Tensor, sampling_rate: float, window: float, step: float,
                lengths: Optional[torch.Tensor] = None, dtype: torch.dtype = _F32) -> torch.Tensor:
    """Spectrogram rows [B, R, window // 2] of ``batch.spectrogram_batch``."""
    return batch.spectrogram_batch(signals.contiguous(), sampling_rate, window, step, lengths=_c(lengths), dtype=dtype)


@spectrogram.register_fake
def _(signals, sampling_rate, window, step, lengths=None, dtype=_F32):
    _check_dtype(dtype)
    B, N = _clip_shape(signals)
    w, s = _plan_args(window, step)
    R, refused = spectrogram_rows(N, w, s)
    if refused:
        _refuse(_lib.ERR_TOO_SHORT)
    return signals.new_empty((B, R, w // 2), dtype=dtype)


@torch.library.custom_op("b200aa::chromagram", mutates_args=(), device_types="cuda")
def chromagram(signals: torch.Tensor, sampling_rate: float, window: float, step: float,
               lengths: Optional[torch.Tensor] = None, dtype: torch.dtype = _F32) -> torch.Tensor:
    """Chromagram rows [B, R, 12] of ``batch.chromagram_batch``."""
    return batch.chromagram_batch(signals.contiguous(), sampling_rate, window, step, lengths=_c(lengths), dtype=dtype)


@chromagram.register_fake
def _(signals, sampling_rate, window, step, lengths=None, dtype=_F32):
    _check_dtype(dtype)
    B, N = _clip_shape(signals)
    w, s = _plan_args(window, step)
    R, refused = chromagram_rows(N, w, s)
    if R <= 0 or (lengths is None and N - s - w < 0):
        _refuse(_lib.ERR_TOO_SHORT)
    if lengths is None and refused and B != 0:
        _refuse(_lib.ERR_INVALID)           # a clipped last frame shorter than window / 2
    return signals.new_empty((B, R, 12), dtype=dtype)


@torch.library.custom_op("b200aa::frame_counts", mutates_args=(), device_types="cuda")
def frame_counts(lengths: torch.Tensor, window: float, step: float, step_ratio: int = 1) -> Tuple[torch.Tensor, torch.Tensor]:
    """(n_frames, n_windows) int64 [B] of ``batch.frame_counts``: each clip's short-term frames and mid-term windows."""
    return batch.frame_counts(lengths.contiguous(), window, step, step_ratio)


@frame_counts.register_fake
def _(lengths, window, step, step_ratio=1):
    if lengths.dim() != 1:
        raise ValueError("lengths must be a tensor [B]")
    if step_ratio < 1:
        raise ValueError("mid-term step shorter than half a short-term step")
    if (int(window) < 1 or int(step) < 1) and lengths.shape[0] != 0:
        _refuse(_lib.ERR_INVALID)
    return lengths.new_empty(lengths.shape, dtype=torch.int64), lengths.new_empty(lengths.shape, dtype=torch.int64)


@torch.library.custom_op("b200aa::row_counts", mutates_args=(), device_types="cuda")
def row_counts(lengths: torch.Tensor, window: float, step: float, which: int) -> torch.Tensor:
    """Per-clip rows int64 [B] of a ragged spectrogram (``which = 0``) or chromagram (``which = 1``), ``batch.row_counts``."""
    return batch.row_counts(lengths.contiguous(), window, step, which)


@row_counts.register_fake
def _(lengths, window, step, which):
    if lengths.dim() != 1:
        raise ValueError("lengths must be a tensor [B]")
    if which not in (0, 1):
        raise ValueError("which must be 0 (spectrogram) or 1 (chromagram)")
    if (int(window) < 1 or int(step) < 1) and lengths.shape[0] != 0:
        _refuse(_lib.ERR_INVALID)
    return lengths.new_empty(lengths.shape, dtype=torch.int64)


@torch.library.custom_op("b200aa::mid_pool", mutates_args=(), device_types="cuda")
def mid_pool(st: torch.Tensor, ratio: int, step_ratio: int, n_frames: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Mid-term mean / std pooling [B, 2F, M] of ``batch.mid_pool_batch``, in the rows' dtype."""
    return batch.mid_pool_batch(st.contiguous(), ratio, step_ratio, n_frames=_c(n_frames), dtype=st.dtype)


@mid_pool.register_fake
def _(st, ratio, step_ratio, n_frames=None):
    B, F, T = _rows_arg(st)
    if step_ratio < 1 or (n_frames is None and T < 1):
        _refuse(_lib.ERR_INVALID)
    return st.new_empty((B, 2 * F, mid_windows(T, step_ratio)))


@torch.library.custom_op("b200aa::mid_feature_extraction", mutates_args=(), device_types="cuda")
def mid_feature_extraction(signals: torch.Tensor, sampling_rate: float, mid_window: float, mid_step: float,
                           short_window: float, short_step: float, lengths: Optional[torch.Tensor] = None,
                           dtype: torch.dtype = _F32) -> Tuple[torch.Tensor, torch.Tensor]:
    """(mid [B, 136, M], st [B, 68, T]) of ``batch.mid_feature_extraction_batch``."""
    return batch.mid_feature_extraction_batch(signals.contiguous(), sampling_rate, mid_window, mid_step, short_window,
                                              short_step, lengths=_c(lengths), dtype=dtype)


@mid_feature_extraction.register_fake
def _(signals, sampling_rate, mid_window, mid_step, short_window, short_step, lengths=None, dtype=_F32):
    _check_dtype(dtype)
    B, N = _clip_shape(signals)
    T = _frames_or_refuse(N, short_window, short_step)
    _, stepr = batch.mid_ratios(mid_window, mid_step, short_window, short_step)
    if stepr < 1:
        raise ValueError("mid-term step shorter than half a short-term step")
    st = signals.new_empty((B, 68, T), dtype=dtype)
    return signals.new_empty((B, 136, mid_windows(T, stepr)), dtype=dtype), st


@torch.library.custom_op("b200aa::long_term_mean", mutates_args=(), device_types="cuda")
def long_term_mean(mid: torch.Tensor, n_windows: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Mean over the mid-term windows [B, rows] of ``batch.long_term_mean_batch``, in the rows' dtype."""
    return batch.long_term_mean_batch(mid.contiguous(), _c(n_windows))


@long_term_mean.register_fake
def _(mid, n_windows=None):
    B, rows, M = _rows_arg(mid)
    if n_windows is None and M < 1:
        _refuse(_lib.ERR_INVALID)
    return mid.new_empty((B, rows))


@torch.library.custom_op("b200aa::beat_extraction", mutates_args=(), device_types="cuda")
def beat_extraction(st: torch.Tensor, window_size: float, n_frames: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(bpm, ratio) float64 [B, 2] of ``batch.beat_extraction_batch`` on float32 or float64 rows."""
    return batch.beat_extraction_batch(st.contiguous(), window_size, n_frames=_c(n_frames), dtype=st.dtype)


@beat_extraction.register_fake
def _(st, window_size, n_frames=None):
    B, _, _ = _rows_arg(st, 19)
    if round(2.0 / window_size) < 1:
        raise ValueError("round(2 / window_size) = %d: the beat histogram needs at least one bin" % round(2.0 / window_size))
    return st.new_empty((B, 2), dtype=torch.float64)


OPS = ("clip_stats", "feature_extraction", "spectrogram", "chromagram", "frame_counts", "row_counts", "mid_pool",
       "mid_feature_extraction", "long_term_mean", "beat_extraction")
