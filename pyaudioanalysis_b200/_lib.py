"""ctypes binding of libb200aa.so (the C ABI declared in include/b200aa.h).

There is no CPU fallback: if the library is missing or the device is not an H100-class (sm_90) GPU the
calls raise.  The library itself is pure C ABI; torch is only used by callers for device memory.
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200AA_LIB") or os.path.join(_HERE, "libb200aa.so")   # override: A/B builds only

OK = 0
ERR_INVALID, ERR_TOO_SHORT, ERR_CHROMA, ERR_MEL_RANGE, ERR_CUDA, ERR_UNSUPPORTED, ERR_NO_DEVICE = -1, -2, -3, -4, -5, -6, -7
DTYPE_I16, DTYPE_F32, DTYPE_F64 = 0, 1, 2

_lib = None
_lock = threading.Lock()

c_i64 = ctypes.c_int64
c_vp = ctypes.c_void_p
c_int = ctypes.c_int

# name -> (restype, argtypes); must list every symbol include/b200aa.h declares
SIGNATURES = {
    "b200aa_abi_version": (c_int, []),
    "b200aa_status_string": (ctypes.c_char_p, [c_int]),
    "b200aa_last_cuda_error": (ctypes.c_char_p, []),
    "b200aa_device_ok": (c_int, []),
    "b200aa_host_table": (c_int, [c_int, c_int, c_int, c_vp]),
    "b200aa_num_frames": (c_i64, [c_i64, c_int, c_int]),
    "b200aa_spectrogram_rows": (c_i64, [c_i64, c_int, c_int]),
    "b200aa_chromagram_rows": (c_i64, [c_i64, c_int, c_int]),
    "b200aa_mid_windows": (c_i64, [c_i64, c_int]),
    "b200aa_plan_create": (c_int, [ctypes.POINTER(c_vp), c_int, c_int, c_int]),
    "b200aa_plan_destroy": (None, [c_vp]),
    "b200aa_plan_kernel_kind": (c_int, [c_vp]),
    "b200aa_plan_force_generic": (c_int, [c_vp, c_int]),
    "b200aa_plan_prefer_kernel": (c_int, [c_vp, c_int]),
    "b200aa_plan_trim": (c_int, [c_vp]),
    "b200aa_debug_set_dump": (c_int, [c_vp]),
    "b200aa_clip_stats": (c_int, [c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "b200aa_st_features": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_int, c_vp, c_i64, c_vp]),
    "b200aa_spectrogram": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "b200aa_chromagram": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp]),
    # (plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream)
    "b200aa_spectrogram_ragged": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "b200aa_chromagram_ragged": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp]),
    # (d_len, n_clips, window, step, which: 0 spectrogram / 1 chromagram, d_rows, stream)
    "b200aa_row_counts": (c_int, [c_vp, c_i64, c_int, c_int, c_int, c_vp, c_vp]),
    "b200aa_mid_pool": (c_int, [c_vp, c_i64, c_int, c_i64, c_i64, c_int, c_int, c_vp, c_vp]),
    "b200aa_long_term_mean": (c_int, [c_vp, c_i64, c_int, c_i64, c_vp, c_vp]),
    "b200aa_frame_counts": (c_int, [c_vp, c_i64, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "b200aa_mid_pool_ragged": (c_int, [c_vp, c_i64, c_int, c_i64, c_vp, c_int, c_int, c_vp, c_vp]),
    "b200aa_long_term_mean_ragged": (c_int, [c_vp, c_i64, c_int, c_i64, c_vp, c_vp, c_vp]),
    "b200aa_normalize_windows": (c_int, [c_vp, c_i64, c_int, c_i64, c_vp, c_vp, c_vp, c_vp]),
    # (d_arena, arena_bytes, h_clips, n_clips, out_dtype, d_out, n_out, out_stride, stream)
    "b200aa_decode_pcm": (c_int, [c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_i64, c_i64, c_vp]),
    "b200aa_beat_extraction": (c_int, [c_vp, c_i64, c_int, c_i64, c_i64, c_vp, ctypes.c_double, c_vp, c_vp]),
    # (d_feats, d_slots, n_train, n_feats, n_classes, k, d_query, dtype, n_query, q_stride, d_ids, d_P, stream)
    "b200aa_knn_classify": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_i64, c_vp, c_int, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "b200aa_st_features_host": (c_int, [c_vp, c_vp, c_int, c_i64, c_i64, c_int, c_vp]),
    "b200aa_spectrogram_host": (c_int, [c_vp, c_vp, c_int, c_i64, c_vp]),
    "b200aa_chromagram_host": (c_int, [c_vp, c_vp, c_int, c_i64, c_vp]),
    "b200aa_mid_features_host": (c_int, [c_vp, c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp]),
    "b200aa_host_alloc": (c_int, [ctypes.POINTER(c_vp), ctypes.c_size_t]),
    "b200aa_host_free": (c_int, [c_vp]),
    "b200aa_peer_buffer_create": (c_int, [ctypes.c_size_t, ctypes.POINTER(c_vp), c_vp]),
    "b200aa_peer_buffer_open": (c_int, [c_vp, ctypes.POINTER(c_vp)]),
    "b200aa_peer_copy": (c_int, [c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200aa_peer_buffer_close": (c_int, [c_vp, c_int]),
    "b200aa_launch_count": (c_i64, []),
}


def lib():
    """Load libb200aa.so (once).  Raises if it has not been built -- there is no fallback."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        "libb200aa.so is missing (%s); build it with `python -m pyaudioanalysis_b200.build` "
                        "-- this package has no CPU fallback" % LIB_PATH)
                L = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in SIGNATURES.items():
                    fn = getattr(L, name)
                    fn.restype = res
                    fn.argtypes = args
                if L.b200aa_abi_version() != 1:
                    raise RuntimeError("libb200aa.so ABI version mismatch")
                _lib = L
    return _lib


def check(status):
    """Map a b200aa_status to the exception the reference would raise (or RuntimeError)."""
    if status == OK:
        return
    L = lib()
    text = L.b200aa_status_string(status).decode()
    if status in (ERR_TOO_SHORT, ERR_CHROMA, ERR_INVALID):
        raise ValueError(text)          # ShortTermFeatures.py:684 / :290-294 raise ValueError
    if status == ERR_MEL_RANGE:
        raise IndexError(text)          # ShortTermFeatures.py:230-231 raises IndexError
    if status == ERR_CUDA:
        raise RuntimeError(text + ": " + L.b200aa_last_cuda_error().decode())
    raise RuntimeError(text)


class Plan:
    """RAII wrapper of b200aa_plan (constant tables of one (fs, window, step) on the current device)."""

    def __init__(self, fs, window, step):
        self.fs, self.window, self.step = int(fs), int(window), int(step)
        self.K = self.window // 2
        h = c_vp()
        check(lib().b200aa_plan_create(ctypes.byref(h), self.fs, self.window, self.step))
        self.handle = h

    def kernel_kind(self):
        return lib().b200aa_plan_kernel_kind(self.handle)

    def force_generic(self, on=True):
        return lib().b200aa_plan_force_generic(self.handle, 1 if on else 0)

    def prefer_kernel(self, kind):
        """-1 automatic, 0 generic, 1 register-tiled CTA kernel, 2 warp-autonomous pair kernel, 3 warp-autonomous per-frame
        kernel (testing / A-B)."""
        check(lib().b200aa_plan_prefer_kernel(self.handle, int(kind)))
        return self

    def trim(self):
        """Free the device workspaces the host entry points keep between calls."""
        check(lib().b200aa_plan_trim(self.handle))

    def __del__(self):
        try:
            if getattr(self, "handle", None) and _lib is not None:
                _lib.b200aa_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


import collections

_plans = collections.OrderedDict()
_plans_lock = threading.Lock()
MAX_CACHED_PLANS = 32       # least recently used plans beyond this are dropped (their device tables and workspaces are freed)


def get_plan(fs, window, step, device=None):
    """Plans are cached per (device, fs, window, step), least recently used first out."""
    if device is None:
        try:
            import torch
            device = torch.cuda.current_device() if torch.cuda.is_available() else 0
        except Exception:
            device = 0
    key = (int(device), int(fs), int(window), int(step))
    with _plans_lock:
        pl = _plans.get(key)
        if pl is None:
            pl = Plan(fs, window, step)
            _plans[key] = pl
            while len(_plans) > MAX_CACHED_PLANS:
                _plans.popitem(last=False)          # Plan.__del__ destroys it once no caller holds it any more
        else:
            _plans.move_to_end(key)
        return pl


def host_table(fs, window, which):
    """Dense host tables (float64): which = 'mel' [40,K], 'chroma' [12,K], 'dct' [13,40]."""
    import numpy as np
    K = int(window) // 2
    idx = {"mel": 0, "chroma": 1, "dct": 2}[which]
    shape = {0: (40, K), 1: (12, K), 2: (13, 40)}[idx]
    out = np.zeros(shape, dtype=np.float64)
    check(lib().b200aa_host_table(int(fs), int(window), idx, out.ctypes.data_as(c_vp)))
    return out
