"""H100-native drop-in for pyAudioAnalysis' short-term / mid-term feature path.

    from pyaudioanalysis_b200 import ShortTermFeatures, MidTermFeatures

mirror ``pyAudioAnalysis.ShortTermFeatures.{feature_extraction, spectrogram, chromagram}`` and
``pyAudioAnalysis.MidTermFeatures.mid_feature_extraction`` (same names, arguments, return
values and error behaviour) on top of hand-written sm_90a CUDA (``libb200aa.so``, C ABI in
``include/b200aa.h``).  ``install()`` rebinds those attributes on an imported pyAudioAnalysis.
There is no CPU fallback.
"""
from . import ShortTermFeatures, MidTermFeatures, consumers  # noqa: F401
from .batch import (feature_extraction_batch, mid_feature_extraction_batch, clip_stats,  # noqa: F401
                    spectrogram_batch, chromagram_batch, beat_extraction_batch, frame_counts, mid_pool_batch,
                    long_term_mean_batch, row_counts)
from .audioio import load_batch  # noqa: F401
from .install import install, uninstall  # noqa: F401

__all__ = ["ShortTermFeatures", "MidTermFeatures", "consumers", "feature_extraction_batch", "mid_feature_extraction_batch",
           "spectrogram_batch", "chromagram_batch", "beat_extraction_batch", "frame_counts", "mid_pool_batch",
           "long_term_mean_batch", "row_counts", "clip_stats", "load_batch", "install", "uninstall"]
