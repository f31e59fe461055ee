"""Batched device API: [B, N] clips resident in HBM -> feature tensors resident in HBM.

torch supplies device memory and the current stream; every operation is a C-ABI call into
libb200aa.so (hand-written sm_90a kernels).  Nothing here computes on the CPU.
"""
import ctypes

import torch

from . import _lib
from ._lib import lib, check, get_plan, DTYPE_I16, DTYPE_F32

NORM_BYTES = 32


class DeviceBuffer:
    """Raw float32 device memory [shape] given by address -- e.g. a window of another GPU's HBM mapped over NVLink
    (dist.PeerGather).  Accepted as ``out=`` of feature_extraction_batch; the caller guarantees size and lifetime."""

    def __init__(self, ptr, shape):
        self.ptr, self.shape, self.is_cuda = int(ptr), tuple(int(s) for s in shape), True

    def data_ptr(self):
        return self.ptr


def _require_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("%s must be a CUDA tensor (there is no CPU fallback)" % name)


def _dtype_code(t):
    if t.dtype == torch.int16:
        return DTYPE_I16
    if t.dtype == torch.float32:
        return DTYPE_F32
    raise TypeError("clips must be int16 or float32, got %s" % t.dtype)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _prep(signals, lengths):
    _require_cuda(signals, "signals")
    if signals.dim() == 1:
        signals = signals.unsqueeze(0)
    if signals.dim() != 2 or signals.stride(1) != 1:
        raise ValueError("signals must be [B, N] with contiguous samples")
    B, N = signals.shape
    stride = signals.stride(0) if B > 1 else N
    if stride < N:
        raise ValueError("overlapping clips are not supported")
    len_ptr = None
    if lengths is not None:
        _require_cuda(lengths, "lengths")
        lengths = lengths.to(torch.int64).contiguous()
        if lengths.numel() != B:
            raise ValueError("lengths must have one entry per clip")
        len_ptr = ctypes.c_void_p(lengths.data_ptr())
    return signals, B, N, stride, lengths, len_ptr


def clip_stats(signals, lengths=None, out=None):
    """Per-clip normalisation records (kernel 0).  Returns a uint8 CUDA tensor [B, 32]."""
    signals, B, N, stride, lengths, len_ptr = _prep(signals, lengths)
    with torch.cuda.device(signals.device):
        norm = out if out is not None else torch.empty((B, NORM_BYTES), dtype=torch.uint8, device=signals.device)
        check(lib().b200aa_clip_stats(ctypes.c_void_p(signals.data_ptr()), _dtype_code(signals), B, N, stride,
                                      len_ptr, ctypes.c_void_p(norm.data_ptr()), _stream()))
    return norm


def feature_extraction_batch(signals, sampling_rate, window, step, deltas=True, out=None, lengths=None, norm=None,
                             plan=None):
    """Short-term features of B clips: CUDA [B, N] int16/float32 -> CUDA float32 [B, 68|34, T].

    Same semantics per clip as ShortTermFeatures.feature_extraction (reference
    ShortTermFeatures.py:543-685); ``lengths`` (int64 CUDA [B]) allows ragged clips: columns
    beyond a clip's own frame count are left as they are in ``out`` (zeros if allocated here).
    """
    window, step = int(window), int(step)
    signals, B, N, stride, lengths, len_ptr = _prep(signals, lengths)
    F = 68 if deltas else 34
    with torch.cuda.device(signals.device):
        plan = plan or get_plan(sampling_rate, window, step, signals.device.index)
        T = lib().b200aa_num_frames(N, window, step)
        if T <= 0:
            check(_lib.ERR_TOO_SHORT)
        if out is None:
            alloc = torch.zeros if lengths is not None else torch.empty
            out = alloc((B, F, T), dtype=torch.float32, device=signals.device)
        elif isinstance(out, DeviceBuffer):
            if out.shape[0] != B or out.shape[1] != F or out.shape[2] < T:
                raise ValueError("out must be float32 [B, %d, >=%d]" % (F, T))
        else:
            _require_cuda(out, "out")
            if out.dtype != torch.float32 or out.shape[0] != B or out.shape[1] != F or out.shape[2] < T or not out.is_contiguous():
                raise ValueError("out must be contiguous float32 [B, %d, >=%d]" % (F, T))
        if norm is None:
            norm = clip_stats(signals, lengths)
        check(lib().b200aa_st_features(plan.handle, ctypes.c_void_p(signals.data_ptr()), _dtype_code(signals), B, N, stride,
                                       len_ptr, ctypes.c_void_p(norm.data_ptr()), 1 if deltas else 0,
                                       ctypes.c_void_p(out.data_ptr()), out.shape[2], _stream()))
    return out


def _counts(t, B, name):
    """A per-clip count argument: an int64 CUDA tensor [B]."""
    _require_cuda(t, name)
    if t.dtype != torch.int64 or tuple(t.shape) != (B,):
        raise ValueError("%s must be an int64 tensor [B]" % name)
    return t.contiguous()


def frame_counts(lengths, window, step, step_ratio=None):
    """Per-clip counts of a ragged batch, computed on the device: int64 CUDA ``n_frames [B]`` (short-term frames of
    ``lengths[b]`` samples, ``feature_extraction_batch``'s columns of clip b), and with ``step_ratio`` also
    ``n_windows [B]`` (its mid-term windows, ``mid_pool_batch``'s columns) as ``(n_frames, n_windows)``."""
    _require_cuda(lengths, "lengths")
    if lengths.dim() != 1:
        raise ValueError("lengths must be a tensor [B]")
    lengths = lengths.to(torch.int64).contiguous()
    B = lengths.shape[0]
    with torch.cuda.device(lengths.device):
        frames = torch.empty((B,), dtype=torch.int64, device=lengths.device)
        windows = None if step_ratio is None else torch.empty((B,), dtype=torch.int64, device=lengths.device)
        if step_ratio is not None and int(step_ratio) < 1:
            raise ValueError("mid-term step shorter than half a short-term step")
        if B:
            check(lib().b200aa_frame_counts(ctypes.c_void_p(lengths.data_ptr()), B, int(window), int(step),
                                            1 if step_ratio is None else int(step_ratio), ctypes.c_void_p(frames.data_ptr()),
                                            None if windows is None else ctypes.c_void_p(windows.data_ptr()), _stream()))
    return frames if windows is None else (frames, windows)


def mid_pool_batch(st, ratio, step_ratio, n_frames=None):
    """Mean / population-std pooling (kernel 2): CUDA float32 [B, F, T] -> [B, 2F, M].

    ``n_frames``: None (every clip has T frames), an int (every clip has that many), or an int64 CUDA tensor [B] of each
    clip's own frame count, clamped to [0, T], e.g. from ``frame_counts``.  With a tensor the output is zero-filled
    [B, 2F, mid_windows(T)] and clip b's first M_b = mid_windows(n_frames[b]) columns are bit for bit what the clip gives
    pooled alone with ``n_frames = n_frames[b]``."""
    _require_cuda(st, "st")
    if st.dim() != 3 or st.dtype != torch.float32 or not st.is_contiguous():
        raise ValueError("st must be contiguous float32 [B, F, T]")
    B, F, Tst = st.shape
    if isinstance(n_frames, torch.Tensor):
        n_frames = _counts(n_frames, B, "n_frames")
        if int(step_ratio) < 1:
            check(_lib.ERR_INVALID)
        M = lib().b200aa_mid_windows(Tst, int(step_ratio))
        with torch.cuda.device(st.device):
            mid = torch.zeros((B, 2 * F, M), dtype=torch.float32, device=st.device)
            if mid.numel():
                check(lib().b200aa_mid_pool_ragged(ctypes.c_void_p(st.data_ptr()), B, F, Tst,
                                                   ctypes.c_void_p(n_frames.data_ptr()), int(ratio), int(step_ratio),
                                                   ctypes.c_void_p(mid.data_ptr()), _stream()))
        return mid
    T = Tst if n_frames is None else int(n_frames)
    M = lib().b200aa_mid_windows(T, int(step_ratio))
    with torch.cuda.device(st.device):
        mid = torch.empty((B, 2 * F, M), dtype=torch.float32, device=st.device)
        check(lib().b200aa_mid_pool(ctypes.c_void_p(st.data_ptr()), B, F, T, Tst, int(ratio), int(step_ratio),
                                    ctypes.c_void_p(mid.data_ptr()), _stream()))
    return mid


def long_term_mean_batch(mid, n_windows=None):
    """Mean over the mid-term windows: CUDA float32 [B, rows, M] -> [B, rows] (MidTermFeatures.py:200-201).

    ``n_windows`` (int64 CUDA [B], entries clamped to [0, M]): clip b averages its first n_windows[b] columns, bit for
    bit as it would alone; a clip of no windows gives NaN, as np.mean of an empty axis does."""
    _require_cuda(mid, "mid")
    if mid.dim() != 3 or mid.dtype != torch.float32 or not mid.is_contiguous():
        raise ValueError("mid must be contiguous float32 [B, rows, M]")
    B, rows, M = mid.shape
    with torch.cuda.device(mid.device):
        out = torch.empty((B, rows), dtype=torch.float32, device=mid.device)
        if n_windows is None:
            check(lib().b200aa_long_term_mean(ctypes.c_void_p(mid.data_ptr()), B, rows, M, ctypes.c_void_p(out.data_ptr()),
                                              _stream()))
            return out
        n_windows = _counts(n_windows, B, "n_windows")
        if M == 0:                  # no columns to read: give the kernel a valid pointer, every clip averages none
            mid = mid.new_zeros((1,))
        check(lib().b200aa_long_term_mean_ragged(ctypes.c_void_p(mid.data_ptr()), B, rows, M,
                                                 ctypes.c_void_p(n_windows.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                                 _stream()))
    return out


def beat_extraction_batch(st, window_size, n_frames=None):
    """Beat rate of every clip (kernel 4): CUDA float32 [B, F >= 19, T] short-term features -> CUDA float64 [B, 2] of
    (bpm, ratio), bit for bit ``MidTermFeatures.beat_extraction(st[b, :, :n_frames[b]], window_size)`` on the same values
    widened to float64.  ``n_frames`` (int64 CUDA [B], entries clamped to [0, T]) gives each clip's own frame count in a
    ragged batch, e.g. the frame counts of ``feature_extraction_batch(..., lengths=)``'s clips.  ``window_size`` is the
    short-term step in seconds, as in the reference; round(2 / window_size) < 1 raises ValueError like the host function."""
    _require_cuda(st, "st")
    if st.dim() != 3 or st.dtype != torch.float32 or not st.is_contiguous() or st.shape[1] < 19:
        raise ValueError("st must be contiguous float32 [B, F >= 19, T]")
    max_beat_time = round(2.0 / window_size)
    if max_beat_time < 1:
        raise ValueError("round(2 / window_size) = %d: the beat histogram needs at least one bin" % max_beat_time)
    B, F, T = st.shape
    fr_ptr = None
    if n_frames is not None:
        n_frames = _counts(n_frames, B, "n_frames")
        fr_ptr = ctypes.c_void_p(n_frames.data_ptr())
    with torch.cuda.device(st.device):
        out = torch.empty((B, 2), dtype=torch.float64, device=st.device)
        if B == 0:
            return out
        if T == 0:                  # no frames has an answer too, (60 / window, NaN); give the kernel a valid pointer
            st, T, fr_ptr = st.new_zeros((B, F, 1)), 0, None
        check(lib().b200aa_beat_extraction(ctypes.c_void_p(st.data_ptr()), B, F, T, T, fr_ptr, float(window_size),
                                           ctypes.c_void_p(out.data_ptr()), _stream()))
    return out


def mid_ratios(mid_window, mid_step, short_window, short_step):
    """MidTermFeatures.py:100-102 (Python round(): half to even).  window/step truncation happens
    inside feature_extraction only (ShortTermFeatures.py:563-564); the ratios use the raw arguments."""
    ratio = round((mid_window - (short_window - short_step)) / short_step)
    stepr = int(round(mid_step / short_step))
    return int(ratio), stepr


def mid_feature_extraction_batch(signals, sampling_rate, mid_window, mid_step, short_window, short_step, lengths=None):
    """Batched MidTermFeatures.mid_feature_extraction: returns (mid [B,136,M], st [B,68,T]) on the GPU.  ``ratio <= 0``
    pools Python slices as the reference does (empty windows give 0); a step ratio < 1 raises ValueError.
    ``lengths`` (int64 CUDA [B]) makes the batch ragged: clip b is ``signals[b, :lengths[b]]``, its columns past its own
    frame count in ``st`` and past its own window count in ``mid`` are zero (``frame_counts`` gives both counts)."""
    st = feature_extraction_batch(signals, sampling_rate, short_window, short_step, deltas=True, lengths=lengths)
    ratio, stepr = mid_ratios(mid_window, mid_step, short_window, short_step)
    if stepr < 1:
        raise ValueError("mid-term step shorter than half a short-term step")
    n_frames = None if lengths is None else frame_counts(lengths, short_window, short_step)
    return mid_pool_batch(st, ratio, stepr, n_frames=n_frames), st


def row_counts(lengths, window, step, which):
    """Per-clip output rows of a ragged ``spectrogram_batch`` (``which = 0``) or ``chromagram_batch`` (``which = 1``),
    computed on the device: int64 CUDA [B], ``lengths[b]``'s row count, or 0 for a clip the equal-length call refuses
    (every accepted clip has at least one row)."""
    _require_cuda(lengths, "lengths")
    if lengths.dim() != 1:
        raise ValueError("lengths must be a tensor [B]")
    if which not in (0, 1):
        raise ValueError("which must be 0 (spectrogram) or 1 (chromagram)")
    lengths = lengths.to(torch.int64).contiguous()
    B = lengths.shape[0]
    with torch.cuda.device(lengths.device):
        rows = torch.empty((B,), dtype=torch.int64, device=lengths.device)
        if B:
            check(lib().b200aa_row_counts(ctypes.c_void_p(lengths.data_ptr()), B, int(window), int(step), which,
                                          ctypes.c_void_p(rows.data_ptr()), _stream()))
    return rows


def spectrogram_batch(signals, sampling_rate, window, step, plan=None, norm=None, out=None, lengths=None):
    """CUDA [B, N] -> CUDA float32 [B, R, K] (ShortTermFeatures.py:389-452 rows, per clip).  ``norm``: records of a previous
    ``clip_stats`` call on the same clips; ``out``: a contiguous float32 [B, R, K] tensor to write into.  ``lengths``
    (int64 CUDA [B]) makes the batch ragged: clip b is ``signals[b, :lengths[b]]``, R is the row count of N samples, and
    only clip b's first ``row_counts(lengths, window, step, 0)[b]`` rows are written, bit for bit what the clip gives
    alone (none for a clip the equal-length call refuses); an output allocated here is zero-filled."""
    window, step = int(window), int(step)
    signals, B, N, stride, lengths, len_ptr = _prep(signals, lengths)
    with torch.cuda.device(signals.device):
        plan = plan or get_plan(sampling_rate, window, step, signals.device.index)
        R = lib().b200aa_spectrogram_rows(N, window, step)
        if R <= 0:
            check(_lib.ERR_TOO_SHORT)
        if out is None:
            alloc = torch.zeros if lengths is not None else torch.empty
            out = alloc((B, R, window // 2), dtype=torch.float32, device=signals.device)
        elif tuple(out.shape) != (B, R, window // 2) or out.dtype != torch.float32 or not out.is_contiguous() or not out.is_cuda:
            raise ValueError("out must be a contiguous float32 CUDA tensor [B, %d, %d]" % (R, window // 2))
        if norm is None:
            norm = clip_stats(signals, lengths)
        args = (plan.handle, ctypes.c_void_p(signals.data_ptr()), _dtype_code(signals), B, N, stride)
        tail = (ctypes.c_void_p(norm.data_ptr()), ctypes.c_void_p(out.data_ptr()), _stream())
        if lengths is None:
            check(lib().b200aa_spectrogram(*args, *tail))
        else:
            check(lib().b200aa_spectrogram_ragged(*args, len_ptr, *tail))
    return out


def chromagram_batch(signals, sampling_rate, window, step, plan=None, norm=None, lengths=None):
    """CUDA [B, N] -> CUDA float32 [B, R, 12] (ShortTermFeatures.py:324-386 rows, per clip).  ``lengths`` (int64 CUDA [B])
    makes the batch ragged: clip b is ``signals[b, :lengths[b]]``, R is the row count of N samples, and the output is
    zero-filled; clip b's first ``row_counts(lengths, window, step, 1)[b]`` rows are bit for bit what the clip gives alone,
    clipped last frames included, and a clip the equal-length call refuses keeps zero rows."""
    window, step = int(window), int(step)
    signals, B, N, stride, lengths, len_ptr = _prep(signals, lengths)
    with torch.cuda.device(signals.device):
        plan = plan or get_plan(sampling_rate, window, step, signals.device.index)
        R = lib().b200aa_chromagram_rows(N, window, step)
        if R <= 0 or (lengths is None and N - step - window < 0):
            check(_lib.ERR_TOO_SHORT)
        alloc = torch.zeros if lengths is not None else torch.empty
        out = alloc((B, R, 12), dtype=torch.float32, device=signals.device)
        if norm is None:
            norm = clip_stats(signals, lengths)
        args = (plan.handle, ctypes.c_void_p(signals.data_ptr()), _dtype_code(signals), B, N, stride)
        tail = (ctypes.c_void_p(norm.data_ptr()), ctypes.c_void_p(out.data_ptr()), _stream())
        if lengths is None:
            check(lib().b200aa_chromagram(*args, *tail))
        else:
            check(lib().b200aa_chromagram_ragged(*args, len_ptr, *tail))
    return out
