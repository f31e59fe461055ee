"""Host-buffer pipeline: pinned host clips in, pinned host features out, through the C ABI.

The end-to-end form of the batched API for callers whose audio lives in host memory (the decoded WAV arrays the
reference works on).  ``run`` is ONE call of ``b200aa_st_features_host``: inside the library the batch is cut into
~32 MB chunks and every chunk's H2D copy, kernels and D2H copy are queued on one of three streams, so the transfers
of neighbouring chunks overlap the kernels.  This class only owns the pinned staging buffers (``b200aa_host_alloc``,
allocated after binding the process to the GPU's NUMA node) and validates shapes; no torch in the data path.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import lib, check, get_plan, DTYPE_I16, DTYPE_F32
from . import numa

_NP_CODES = {np.dtype(np.int16): DTYPE_I16, np.dtype(np.float32): DTYPE_F32}


class PinnedArray:
    """A NumPy view of a page-locked host buffer owned by the library (freed with the object)."""

    def __init__(self, shape, dtype):
        self.shape, self.dtype = tuple(int(s) for s in shape), np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = ctypes.c_void_p()
        check(lib().b200aa_host_alloc(ctypes.byref(p), nbytes))
        self._ptr = p
        buf = (ctypes.c_char * max(nbytes, 1)).from_address(p.value) if nbytes else (ctypes.c_char * 1)()
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def __del__(self):
        try:
            if getattr(self, "_ptr", None) is not None and self._ptr.value:
                self.array = None
                lib().b200aa_host_free(self._ptr)
                self._ptr = None
        except Exception:
            pass


class HostPipeline:
    def __init__(self, sampling_rate, window, step, n_samples, max_clips, device=0, deltas=True, dtype=np.int16,
                 bind_numa=True):
        import torch            # device selection only
        self.fs, self.window, self.step, self.n = int(sampling_rate), int(window), int(step), int(n_samples)
        self.deltas = bool(deltas)
        self.F = 68 if deltas else 34
        self.device = int(device)
        self.dtype = np.dtype(dtype)
        if self.dtype not in _NP_CODES:
            raise TypeError("clips must be int16 or float32, got %s" % self.dtype)
        self.T = lib().b200aa_num_frames(self.n, self.window, self.step)
        if self.T <= 0:
            raise ValueError("need at least one array to concatenate")
        self.max_clips = int(max_clips)
        self.numa = numa.bind_to_gpu(self.device) if bind_numa else None
        torch.cuda.set_device(self.device)
        self.plan = get_plan(self.fs, self.window, self.step, self.device)
        self._in = PinnedArray((self.max_clips, self.n), self.dtype)
        self._out = PinnedArray((self.max_clips, self.F, self.T), np.float32)
        self.h_in, self.h_out = self._in.array, self._out.array

    def run(self, host_clips=None, out=None):
        """host_clips: [B, n_samples] NumPy array of the pipeline's dtype (default: the pipeline's own pinned input
        buffer ``h_in``; any other array works, pageable memory just copies slower).  Returns float32 [B, F, T]
        (a view of the pinned ``h_out`` unless ``out`` is given)."""
        x = self.h_in if host_clips is None else host_clips
        if not isinstance(x, np.ndarray):
            x = np.asarray(x.numpy() if hasattr(x, "numpy") else x)
        if x.ndim != 2 or x.shape[1] != self.n or x.shape[0] > self.max_clips or x.shape[0] < 1:
            raise ValueError("host_clips must be [1..%d, %d], got %s" % (self.max_clips, self.n, x.shape))
        if x.dtype != self.dtype:
            raise TypeError("host_clips dtype %s does not match the pipeline's %s (no silent conversion)" % (x.dtype, self.dtype))
        if not x.flags["C_CONTIGUOUS"]:
            raise ValueError("host_clips must be C-contiguous")
        B = x.shape[0]
        dst = self.h_out if out is None else out
        if dst.dtype != np.float32 or dst.shape[0] < B or dst.shape[1:] != (self.F, self.T) or not dst.flags["C_CONTIGUOUS"]:
            raise ValueError("out must be C-contiguous float32 [>=B, %d, %d]" % (self.F, self.T))
        import torch
        with torch.cuda.device(self.device):
            _lib.refuse_capture("b200aa_st_features_host", _lib.HOST_BUFFER_WHY)
            check(lib().b200aa_st_features_host(self.plan.handle, x.ctypes.data_as(ctypes.c_void_p), _NP_CODES[self.dtype], B,
                                                self.n, 1 if self.deltas else 0, dst.ctypes.data_as(ctypes.c_void_p)))
        return dst[:B]
