"""The result contract of the drop-in functions: "float32" (the default) or "float64".

``set_precision("float64")`` makes ``ShortTermFeatures.feature_extraction`` / ``spectrogram`` / ``chromagram``,
``MidTermFeatures.mid_feature_extraction`` and the directory and file wrappers return what the float64 path (kernel 12)
computes -- the reference's float64 arithmetic, within 1e-9 of it -- instead of the float32 path's features widened to
float64.  Read at call time, so callers of the reference reached through ``install()`` follow it.  Process-wide; this
module is the only place it is stored."""
_PRECISIONS = ("float32", "float64")
_precision = "float32"


def set_precision(precision):
    """Choose the drop-ins' result contract: "float32" or "float64"."""
    global _precision
    if precision not in _PRECISIONS:
        raise ValueError("precision must be 'float32' or 'float64', got %r" % (precision,))
    _precision = precision


def get_precision():
    return _precision


def wide():
    """True while the drop-ins return the float64 path's results."""
    return _precision == "float64"


def torch_dtype():
    import torch
    return torch.float64 if wide() else torch.float32
